"""GPU tests of the BS-Roformer separator (`pytest -m gpu`): the rotary gated attention (evk_rope_attn_fwd) at both axis
layouts, the inverse STFT (evk_istft), the band input and row norm kernels and the GELU GEMM epilogue against float64, their
reproducibility and output slices, and BSRoformer.forward / bs_roformer.demix_track against the outputs the reference
computed (tests/golden/bs_roformer.pt, pinned by oracle/pin_bs_roformer.py)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bs_roformer_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "bs_roformer.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
# rel-L2 of the whole net against the fp32 reference.  Measured on an H100: TF32 6.9e-4 / 8.8e-4 (small / full forward),
# 6.3e-4 / 9.4e-4 (demix); 3xTF32 5.5e-6 / 2.0e-5 (forward), 5.1e-6 / 2.1e-5 (demix).  The attention alone reaches 1.1e-5 under
# 3xTF32 at L = 1500 (fp32 softmax sums over 1500 keys), which sets the floor of the precise figures.
TOL_NET, TOL_NET_PRECISE = 2e-3, 6e-5
# evk_rope_attn_fwd against float64, measured on an H100 over the grid below: TF32 at most 9.0e-4 for L <= 62 and 1.35e-3 for
# L in {801, 1500}; 3xTF32 at most 9.9e-7 and 1.1e-5.  The GELU epilogue: TF32 3.1e-4, 3xTF32 4.1e-6 (tolerances 2e-3, 1e-5).
# evk_istft against torch.istft in float64: 1.4e-7 (tolerance 2e-6).
TOL_ATTN, TOL_ATTN_PRECISE = 2e-3, 3e-5


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


@pytest.fixture(scope="module")
def R():
    from easevoice_trainer_b200 import bs_roformer
    return bs_roformer


class _precise:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(1 if self.on else 0)

    def __exit__(self, *exc):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(0)


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a), torch.as_tensor(np.asarray(b) if not torch.is_tensor(b) else b)
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def config(over):
    cfg = dict(O.SHIPPED)
    cfg.update(over)
    return cfg


# ---- rotary gated attention -------------------------------------------------------------------------------------------
def _cs(L):
    c, s = O.rotary_cos_sin(L)
    return torch.stack([c, s], -1).contiguous()


def _attn_ref(X, H, L, layout, cs):
    """float64 on the device: X [B, T, F, ld] packed rows -> [B, T, F, H*64]"""
    D = H * 64
    X = X.double()
    if layout == "time":
        Xs = X.permute(0, 2, 1, 3)                                   # [B, F, T, ld]: sequences (b, f) of length T
    else:
        Xs = X                                                       # [B, T, F, ld]: sequences (b, t) of length F
    n = Xs.shape[0] * Xs.shape[1]
    Xs = Xs.reshape(n, L, -1)
    q, k, v = (Xs[..., i * D:(i + 1) * D].reshape(n, L, H, 64).permute(0, 2, 1, 3) for i in range(3))
    g = Xs[..., 3 * D:3 * D + H].permute(0, 2, 1)
    c, s = cs[:L, :, 0].double().repeat_interleave(2, -1), cs[:L, :, 1].double().repeat_interleave(2, -1)

    def rot(t):
        x = t.unflatten(-1, (-1, 2))
        return t * c + torch.stack((-x[..., 1], x[..., 0]), -1).flatten(-2) * s

    o = torch.softmax(rot(q) @ rot(k).transpose(-1, -2) / 8.0, -1) @ v * torch.sigmoid(g)[..., None]
    o = o.permute(0, 2, 1, 3).reshape(n, L, D)
    if layout == "time":
        return o.reshape(X.shape[0], X.shape[2], L, D).permute(0, 2, 1, 3)
    return o.reshape(X.shape[0], X.shape[1], L, D)


def _run_attn(ops, X, H, L, layout, cs, extra=4):
    B, T, Fb, ld = X.shape
    D = H * 64
    out = torch.full((B * T * Fb, D + extra), 7.0, device=DEV)
    geo = (B, T * Fb, Fb, 1, Fb) if layout == "time" else (B * T, Fb, 1, 0, 1)
    ops.rope_attn(X.view(-1, ld), cs, out[:, :D], H, L, *geo)
    return out


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("H", [2, 8])
@pytest.mark.parametrize("L", [1, 7, 62, 801, 1500])
@pytest.mark.parametrize("layout", ["time", "freq"])
def test_rope_attn_vs_float64(ops, layout, L, H, precise):
    g = torch.Generator().manual_seed(L * 10 + H)
    D = H * 64
    ld = (3 * D + H + 3) // 4 * 4 + 4
    shape = (2, L, 3, ld) if layout == "time" else (1, 3, L, ld)
    X = (torch.randn(shape, generator=g) * 1.5).to(DEV)
    cs = _cs(L).to(DEV)
    with _precise(precise):
        out = _run_attn(ops, X, H, L, layout, cs)
        again = _run_attn(ops, X, H, L, layout, cs)
    assert torch.equal(out, again)                                  # bit-reproducible
    assert (out[:, D:] == 7).all()                                  # nothing outside the output slice is written
    ref = _attn_ref(X, H, L, layout, cs).reshape(-1, D)
    e = rel(out[:, :D], ref)
    print(f"rope_attn {layout} L={L} H={H} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_ATTN_PRECISE if precise else TOL_ATTN), e


# ---- inverse STFT -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft,hop,S", [(2048, 441, 2), (1024, 256, 1), (256, 100, 2), (4096, 1024, 1)])
def test_istft_with_mask_vs_torch(ops, n_fft, hop, S):
    g = torch.Generator().manual_seed(n_fft + hop)
    B, L = 2, 20 * hop + 37
    wav = torch.randn(B * S, L, generator=g).to(DEV)
    cplx = ops.stft(wav, n_fft, hop)
    T, NB = cplx.shape[1], n_fft // 2 + 1
    mask = torch.randn(B * T, 2 * S * NB + 6, generator=g).to(DEV)
    out = ops.istft(cplx, B, S, n_fft, hop, mask=mask[:, :2 * S * NB])
    again = ops.istft(cplx, B, S, n_fft, hop, mask=mask[:, :2 * S * NB])
    assert torch.equal(out, again)
    X = torch.view_as_complex(cplx.double().cpu().contiguous())                          # [B*S, T, NB]
    m = torch.view_as_complex(mask[:, :2 * S * NB].double().cpu().reshape(B, T, NB, S, 2).contiguous())
    m = m.permute(0, 3, 1, 2).reshape(B * S, T, NB)
    ref = torch.istft((X * m).transpose(1, 2), n_fft, hop, n_fft, torch.hann_window(n_fft, dtype=torch.float64))
    assert out.shape == ref.shape
    e = rel(out, ref)
    print(f"istft n_fft={n_fft} hop={hop} S={S} rel-L2 {e:.3g}")
    assert e <= 2e-6, e


def test_istft_output_pitch_and_round_trip(ops):
    n_fft, hop = 2048, 441
    wav = torch.randn(3, 44100, generator=torch.Generator().manual_seed(2)).to(DEV)
    cplx = ops.stft(wav, n_fft, hop)
    n = hop * (cplx.shape[1] - 1)
    buf = torch.full((3, n + 5), 7.0, device=DEV)
    ops.istft(cplx, 3, 1, n_fft, hop, out=buf[:, :n])
    assert (buf[:, n:] == 7).all()
    assert rel(buf[:, :n], wav[:, :n]) <= 1e-6


# ---- band input, row norm, GELU epilogue ------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 2])
def test_band_input_vs_float64(ops, S):
    bands = O.SHIPPED["freqs_per_bands"]
    B, L = 2, 20000
    wav = torch.randn(B * S, L, generator=torch.Generator().manual_seed(S)).to(DEV)
    cplx = ops.stft(wav, 2048, 441)
    T, NB = cplx.shape[1], 1025
    off = torch.tensor(np.concatenate([[0], np.cumsum(bands)]), dtype=torch.int32).to(DEV)
    out = torch.full((B * T, 2 * S * NB + 4), 7.0, device=DEV)
    ops.bs_band_input(cplx, B, S, off, out[:, :2 * S * NB])
    again = out.clone()
    ops.bs_band_input(cplx, B, S, off, again[:, :2 * S * NB])
    assert torch.equal(out, again) and (out[:, 2 * S * NB:] == 7).all()
    x = cplx.double().cpu().reshape(B, S, T, NB, 2).permute(0, 2, 3, 1, 4).reshape(B * T, -1)
    ref = torch.cat([F.normalize(p, dim=-1) for p in x.split([2 * S * f for f in bands], -1)], -1)
    assert rel(out[:, :2 * S * NB], ref) <= 1e-6


def test_row_l2norm_vs_float64(ops):
    x = torch.randn(1000, 520, generator=torch.Generator().manual_seed(4)).to(DEV)
    x[3] = 0
    out = torch.full((1000, 516), 7.0, device=DEV)
    ops.row_l2norm(x[:, :512], out=out[:, :512])
    again = torch.full_like(out, 7.0)
    ops.row_l2norm(x[:, :512], out=again[:, :512])
    assert torch.equal(out, again)                                  # bit-reproducible
    assert (out[:, 512:] == 7).all() and (out[3, :512] == 0).all()
    assert rel(out[:, :512], F.normalize(x[:, :512].double(), dim=-1)) <= 1e-6


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("rows,C,N,c0", [(1000, 512, 2048, 0), (100, 128, 512, 0), (300, 66, 40, 2)])
def test_gelu_epilogue_vs_float64(ops, rows, C, N, c0, precise):
    g = torch.Generator().manual_seed(rows + C)
    xb = torch.randn(rows, C + 4, generator=g).to(DEV)
    w = (torch.randn(N, C, generator=g) / C ** 0.5).to(DEV)
    b = (0.1 * torch.randn(N, generator=g)).to(DEV)
    with _precise(precise):
        pw = ops.pack_weight(w, None, need_pb=False)
        y = torch.full((rows, N + 4), 7.0, device=DEV)
        ops.linear_into(xb[:, c0:c0 + C], pw, y[:, :N], bias=b, act=ops.ACT_GELU)
        y2 = y.clone()
        ops.linear_into(xb[:, c0:c0 + C], pw, y2[:, :N], bias=b, act=ops.ACT_GELU)
    assert torch.equal(y, y2) and (y[:, N:] == 7).all()
    ref = F.gelu(xb[:, c0:c0 + C].double() @ w.double().T + b.double())
    e = rel(y[:, :N], ref)
    print(f"gelu rows={rows} C={C} N={N} precise={precise} rel-L2 {e:.3g}")
    assert e <= (1e-5 if precise else 2e-3), e


# ---- the model --------------------------------------------------------------------------------------------------------
def _model(R, name):
    case = GOLD[name]
    cfg = config(case["over"])
    m = R.BSRoformer(**cfg).to(DEV).load_state_dict(O.init_params(O.param_spec(cfg), case["seed"]))
    return case, m


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "full"])
def test_forward_vs_golden(R, name, precise):
    case, m = _model(R, name)
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    with _precise(precise):
        out = m.forward(raw)
    L = case["fwd_shape"][-1]
    assert out.shape == case["fwd_shape"][:2] + (441 * (L // 441),)
    e = rel(out[..., ::case["stride"]], case["forward"])
    print(f"forward {name} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "full"])
def test_demix_vs_golden(R, name, precise):
    case, m = _model(R, name)
    mix = O.make_audio(case["audio_seed"] + 100, (2, int(case["demix_chunks"] * O.CHUNK)))
    with _precise(precise):
        got = R.demix_track(m, mix, DEV)
    assert list(got) == ["vocals"] and got["vocals"].shape == tuple(mix.shape)
    v = got["vocals"]
    idx = case["demix_idx"].numpy()
    e = rel(v[:, idx], case["demix"])
    print(f"demix {name} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e
    assert np.array_equal(np.nonzero((v == 0).all(0))[0], case["demix_zero"].numpy())


def test_chunk_independent_of_its_launch(R):
    case, m = _model(R, "small")
    a = O.make_audio(5, (3, 2, 44100)).to(DEV)
    both = m.forward(a)
    one = m.forward(a[1:2].contiguous())
    assert torch.equal(both[1:2], one)


def test_max_chunks_1_equals_4(R):
    case, m = _model(R, "small")
    mix = O.make_audio(case["audio_seed"] + 100, (2, int(case["demix_chunks"] * O.CHUNK)))
    a = R.demix_track(m, mix, DEV, max_chunks=1)["vocals"]
    b = R.demix_track(m, mix, DEV, max_chunks=4)["vocals"]
    assert np.array_equal(a, b), float(np.abs(a - b).max())


def test_input_errors_before_any_launch(R, ops):
    case, m = _model(R, "small")
    n0 = ops.launches()
    for bad in (torch.zeros(1, 2, 4096), torch.zeros(1, 1, 4096, device=DEV), torch.zeros(2, 4096, device=DEV),
                torch.zeros(1, 2, 1024, device=DEV)):
        with pytest.raises(ValueError):
            m.forward(bad)
    assert ops.launches() == n0


def test_from_pretrained_checkpoint(R, tmp_path):
    """The documented SeparateMDXC swap: from_pretrained on a reference checkpoint file (fp32, with the rotary_embed.freqs
    entries rotary_embedding_torch saves), then eval() as SeparateMDXC.separate calls it, gives the golden output."""
    case = GOLD["full"]
    P = O.init_params(O.param_spec(O.SHIPPED), case["seed"])
    freqs = O.rotary_inv_freq()
    P.update({k.replace("to_qkv.weight", "rotary_embed.freqs"): freqs.clone() for k in list(P) if k.endswith(".to_qkv.weight")})
    path = tmp_path / "bs_roformer.ckpt"
    torch.save(P, path)
    m = R.BSRoformer.from_pretrained(str(path), device=DEV)
    assert m.eval() is m
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    _, ref = _model(R, "full")
    out = m.forward(raw)
    assert torch.equal(out, ref.forward(raw))
    assert rel(out[..., ::case["stride"]], case["forward"]) <= TOL_NET


def test_load_state_dict_from_cuda_tensors(R):
    """a state_dict loaded with map_location='cuda' folds on the host like a CPU one"""
    case = GOLD["small"]
    cfg = config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    m = R.BSRoformer(**cfg).to(DEV).load_state_dict({k: v.to(DEV) for k, v in P.items()})
    _, ref = _model(R, "small")
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    assert torch.equal(m.forward(raw), ref.forward(raw))
    assert all(v.device.type == "cpu" for v in m.host_w.values()) and all(v.is_cuda for v in m.bias.values())
