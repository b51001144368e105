"""GPU tests of the Mel-Band Roformer separator (`pytest -m gpu`): the overlapping band input (evk_band_input), the averaged
masks (evk_melband_mask_avg) and the RMSNorm with gamma (evk_row_norm) element for element against float64 with the
per-element bounds of tests/cudacore_ref.py, the inverse STFT with an output length (evk_istft) against torch.istft,
and MelBandRoformer.forward / bs_roformer.demix_track against the outputs the reference computed (tests/golden/mel_roformer.pt,
pinned by oracle/pin_mel_roformer.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import mel_roformer_oracle as O
from tests import cudacore_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "mel_roformer.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
SENTINEL = 7.0
# rel-L2 of the whole net against the fp32 reference: TF32 products within the 2e-3 tests/test_gpu_bs_roformer.py holds
# BS-Roformer to, 3xTF32 within 5e-5.  Measured on an H100: TF32 6.7e-4 / 1.52e-3 / 1.08e-3 (small / default / mono forward),
# 6.5e-4 / 1.50e-3 / 1.06e-3 (demix); 3xTF32 6.1e-6 / 3.3e-5 / 3.5e-6 (forward), 6.4e-6 / 3.6e-5 / 4.4e-6 (demix).  The TF32
# error comes mostly from the transformer GEMMs: a CPU emulation of round-to-nearest TF32 operands in every Linear gives
# 9.4e-4 on the mono case, and 5.6e-4 with the transformer Linears exact.
TOL_NET, TOL_NET_PRECISE = 2e-3, 5e-5


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


@pytest.fixture(scope="module")
def M():
    from easevoice_trainer_b200 import mel_band_roformer
    return mel_band_roformer


@pytest.fixture(scope="module")
def BS():
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
    cfg = dict(O.DEFAULT)
    cfg.update(over)
    return cfg


def check(got, ref, what):
    """|got - ref| <= SAFETY * model at every element (bit-exact where the model is 0)"""
    got = got.double().cpu()
    bad = R.outside_gate(got, ref)
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[:6].tolist()
        lines = [f"  {tuple(i)}: got {float(got[tuple(i)])!r} want {float(ref.v[tuple(i)])!r} gate "
                 f"{R.SAFETY * float(ref.e[tuple(i)]):.3g}" for i in idx]
        pytest.fail(f"{what}: {n} of {bad.numel()} outside the gate\n" + "\n".join(lines))


def l2norm_rows(t):
    """E of the kernels' x / max(sqrt(sum x^2), 1e-12) over the last axis: lane-strided partial sums, then warp_sum"""
    C = t.v.shape[-1]
    ss = R.esum(t * t, -1, R.ln_row_chain(C))
    den = R.sqrtf(ss)
    den = E_max(den, 1e-12)
    return t / R.E(den.v[..., None], den.e[..., None])


def E_max(a, floor):
    return R.E(a.v.clamp_min(floor), torch.where(a.v > floor, a.e, torch.zeros_like(a.e)))


# ---- band input, averaged masks, RMSNorm with gamma ---------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("sr,n_fft,nb,hop", [(44100, 2048, 60, 441), (48000, 1024, 24, 256)])
def test_band_input_elementwise(ops, M, S, sr, n_fft, nb, hop):
    bins, band_off, _, _ = M.band_tables(sr, n_fft, nb)
    B, L = 2, 12 * hop + 5
    wav = torch.randn(B * S, L, generator=torch.Generator().manual_seed(S + nb)).to(DEV)
    cplx = ops.stft(wav, n_fft, hop)
    T, W = cplx.shape[1], 2 * S * len(bins)
    dbins, doff = torch.from_numpy(bins).to(DEV), torch.from_numpy(band_off).to(DEV)
    outs = []
    for _ in range(2):
        out = torch.full((B * T, W + 6), SENTINEL, device=DEV)
        ops.band_input(cplx, B, S, doff, dbins, out[:, :W])
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1]) and (outs[0][:, W:] == SENTINEL).all()
    # float64: the same gather ('b t (f s c)' over the bin table), each band's segment normalised
    x = cplx.double().cpu().reshape(B, S, T, -1, 2).permute(0, 2, 3, 1, 4)                 # b t f s c
    x = x[:, :, torch.from_numpy(bins).long()].reshape(B * T, W)
    got = outs[0][:, :W]
    for i in range(nb):
        c0, c1 = 2 * S * band_off[i], 2 * S * band_off[i + 1]
        check(got[:, c0:c1], l2norm_rows(R.E(x[:, c0:c1])), f"band_input band {i} S={S} n_fft={n_fft}")


@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("sr,n_fft,nb", [(44100, 2048, 60), (44100, 512, 8)])
def test_melband_mask_avg_elementwise(ops, M, S, sr, n_fft, nb):
    bins, _, cover, cover_off = M.band_tables(sr, n_fft, nb)
    rows, NB, ns = 301, n_fft // 2 + 1, len(bins)
    g = torch.randn(rows, 2 * S * ns + 2, generator=torch.Generator().manual_seed(nb + S))
    outs = []
    for _ in range(2):
        out = torch.full((rows, 2 * S * NB + 4), SENTINEL, device=DEV)
        ops.melband_mask_avg(g.to(DEV)[:, :2 * S * ns], S, torch.from_numpy(cover_off).to(DEV), torch.from_numpy(cover).to(DEV),
                             out[:, :2 * S * NB])
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1]) and (outs[0][:, 2 * S * NB:] == SENTINEL).all()
    # float64: per (bin, channel, component), 0 + the covering slots in ascending order, then / count
    gs = g[:, :2 * S * ns].double().reshape(rows, ns, S, 2)
    cnt = np.diff(cover_off)
    acc = R.E(torch.zeros(rows, NB, S, 2, dtype=torch.float64))
    for k in range(int(cnt.max())):
        has = torch.from_numpy(cnt > k)
        slot = torch.from_numpy(np.where(cnt > k, cover[np.minimum(cover_off[:-1] + k, ns - 1)], 0)).long()
        term = torch.where(has[None, :, None, None], gs[:, slot], torch.zeros(()))
        acc = acc + R.E(term)
    ref = acc / R.E(torch.from_numpy(cnt).double()[None, :, None, None])
    check(outs[0][:, :2 * S * NB].reshape(rows, NB, S, 2), ref, f"melband_mask_avg S={S} n_fft={n_fft} bands={nb}")
    # bins a single band covers are copied exactly
    one = torch.from_numpy(cnt == 1)
    assert torch.equal(outs[0][:, :2 * S * NB].reshape(rows, NB, S, 2)[:, one].double(),
                       gs[:, torch.from_numpy(cover[cover_off[:-1]]).long()][:, one])


@pytest.mark.parametrize("rows,C,ld", [(1000, 384, 388), (37, 128, 128), (9, 66, 70)])
def test_row_norm_gamma_elementwise(ops, rows, C, ld):
    gen = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, C, generator=gen) * 3.0
    x[3] = 0.0
    gamma = 0.5 + torch.rand(C, generator=gen)
    outs = []
    for _ in range(2):
        xd = torch.full((rows, ld), float("nan"))
        xd[:, :C] = x
        xd = xd.to(DEV)
        out = torch.full((rows, ld), SENTINEL, device=DEV)
        ops.row_norm(xd[:, :C], gamma.to(DEV), out=out[:, :C])
        inplace = xd.clone()
        ops.row_norm(inplace[:, :C], gamma.to(DEV), out=inplace[:, :C])
        outs.append(out.cpu())
        assert torch.equal(inplace[:, :C].cpu(), out[:, :C].cpu())                  # in place gives the same bits
    assert torch.equal(outs[0], outs[1]) and (outs[0][:, C:] == SENTINEL).all()
    assert (outs[0][3, :C] == 0).all()
    scale = float(np.float32(C ** 0.5))
    ref = l2norm_rows(R.E(x.double())) * scale * R.E(gamma.double())
    check(outs[0][:, :C], ref, f"row_norm gamma rows={rows} C={C}")


@pytest.mark.parametrize("n_fft,hop,S,extra", [(2048, 441, 2, 440), (1024, 441, 1, 17), (1024, 256, 1, 0), (256, 100, 2, 99)])
def test_istft_length_vs_torch(ops, n_fft, hop, S, extra):
    g = torch.Generator().manual_seed(n_fft + hop + extra)
    B = 2
    L = 20 * hop + extra
    wav = torch.randn(B * S, L, generator=g).to(DEV)
    cplx = ops.stft(wav, n_fft, hop)
    T, NB = cplx.shape[1], n_fft // 2 + 1
    mask = torch.randn(B * T, 2 * S * NB, generator=g).to(DEV)
    out = torch.full((B * S, L + 3), SENTINEL, device=DEV)
    ops.istft(cplx, B, S, n_fft, hop, mask=mask, out=out[:, :L], length=L)
    assert (out[:, L:] == SENTINEL).all()
    short = ops.istft(cplx, B, S, n_fft, hop, mask=mask)
    assert torch.equal(short, out[:, :hop * (T - 1)])                 # the first hop*(T-1) samples are those of length 0
    X = torch.view_as_complex(cplx.double().cpu().contiguous())
    m = torch.view_as_complex(mask.double().cpu().reshape(B, T, NB, S, 2).contiguous()).permute(0, 3, 1, 2).reshape(B * S, T, NB)
    ref = torch.istft((X * m).transpose(1, 2), n_fft, hop, n_fft, torch.hann_window(n_fft, dtype=torch.float64), length=L)
    e = rel(out[:, :L], ref)
    print(f"istft length n_fft={n_fft} hop={hop} S={S} L={L} rel-L2 {e:.3g}")
    assert e <= 2e-6, e


# ---- the model --------------------------------------------------------------------------------------------------------
def _model(M, name):
    case = GOLD[name]
    cfg = config(case["over"])
    m = M.MelBandRoformer(**cfg).to(DEV).load_state_dict(O.init_params(O.param_spec(cfg), case["seed"]))
    return case, cfg, m


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "default", "mono"])
def test_forward_vs_golden(M, name, precise):
    case, cfg, m = _model(M, name)
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    with _precise(precise):
        out = m.forward(raw)
    assert out.shape == case["fwd_shape"][:2] + (case["forward_len"],)
    e = rel(out[..., ::case["stride"]], case["forward"])
    print(f"forward {name} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "default", "mono"])
def test_demix_vs_golden(M, BS, name, precise):
    case, cfg, m = _model(M, name)
    S = 2 if cfg["stereo"] else 1
    mix = O.make_audio(case["audio_seed"] + 100, (S, int(case["demix_chunks"] * O.CHUNK)))
    with _precise(precise):
        got = BS.demix_track(m, mix, DEV)
    assert list(got) == ["vocals"] and got["vocals"].shape == tuple(mix.shape)
    v = got["vocals"]
    idx = case["demix_idx"].numpy()
    e = rel(v[:, idx], case["demix"])
    print(f"demix {name} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e
    assert np.array_equal(np.nonzero((v == 0).all(0))[0], case["demix_zero"].numpy())


def test_chunk_alone_equals_batched_and_reproducible(M):
    """a chunk's output does not depend on the chunks launched with it, and two runs give the same bits"""
    _, _, m = _model(M, "small")
    a = O.make_audio(5, (4, 2, 44100)).to(DEV)
    four = m.forward(a)
    assert torch.equal(four, m.forward(a))
    assert torch.equal(four[2:3], m.forward(a[2:3].contiguous()))


def test_input_errors_before_any_launch(M, ops):
    _, _, m = _model(M, "small")
    n0 = ops.launches()
    for bad in (torch.zeros(1, 2, 4096), torch.zeros(1, 1, 4096, device=DEV), torch.zeros(2, 4096, device=DEV),
                torch.zeros(1, 2, 1024, device=DEV)):
        with pytest.raises(ValueError):
            m.forward(bad)
    assert ops.launches() == n0


def test_from_pretrained_checkpoint(M):
    """AudioService.uvr5's drop-in: from_pretrained infers the default configuration from the weights of a checkpoint file
    (fp32, with the rotary_embed.freqs entries rotary_embedding_torch saves) and gives the golden output after eval()"""
    import tempfile
    case = GOLD["default"]
    P = O.init_params(O.param_spec(O.DEFAULT), case["seed"])
    freqs = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    P.update({k.replace("to_qkv.weight", "rotary_embed.freqs"): freqs.clone() for k in list(P) if k.endswith(".to_qkv.weight")})
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "mel_band_roformer.ckpt")
        torch.save(P, path)
        m = M.MelBandRoformer.from_pretrained(path, device=DEV)
    assert m.eval() is m
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"]).to(DEV)
    _, _, ref = _model(M, "default")
    out = m.forward(raw)
    assert torch.equal(out, ref.forward(raw))
    assert rel(out[..., ::case["stride"]], case["forward"]) <= TOL_NET
