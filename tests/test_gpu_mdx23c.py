"""GPU tests of the MDX23C separator (`pytest -m gpu`): the 8192-point STFT and iSTFT, the plane instance norm
(evk_instnorm_plane), the 2x2 stride-2 conv, the transposed 2x2 conv, the TDF Linear (evk_mdx_tdf) and the spectral layouts
(evk_mdx_front / evk_mdx_back) element for element against float64, and MDX23C.forward / bs_roformer.demix_track against
the outputs the reference computed (tests/golden/mdx23c.pt, pinned by oracle/pin_mdx23c.py)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mdx23c_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "mdx23c.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
U32 = 2.0 ** -24          # fp32 unit roundoff
U_TF32 = 2.0 ** -11       # TF32 operand rounding (10 explicit mantissa bits, round to nearest)
# rel-L2 of the whole net against the fp32 reference: TF32 products within the roformers' 2e-3, 3xTF32 within 1e-4.  Measured
# on an H100: TF32 1.41e-3 / 1.05e-3 / 1.39e-3 (small / mono / default forward), 1.35e-3 and 1.45e-3 / 1.17e-3 (demix small
# vocals and other / mono); 3xTF32 8.5e-7 / 6.4e-7 / 1.6e-6 (forward), 9.1e-7 / 7.2e-7 (demix).
TOL_NET, TOL_NET_PRECISE = 2e-3, 1e-4


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


@pytest.fixture(scope="module")
def MX():
    from easevoice_trainer_b200 import mdx23c
    return mdx23c


class _precise:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(1 if self.on else 0)

    def __exit__(self, *exc):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(0)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _contraction_bound(absprod, K, precise):
    """per-element bound of a fp32-accumulated sum of K products: operand rounding (TF32: 2 u_tf32 per product; 3xTF32:
    the dropped low x low term, 2^-22 relative) plus the fp32 accumulation (K u32), times the sum of |products|"""
    per = 3 * 2.0 ** -22 if precise else 2 * U_TF32 + U_TF32 ** 2
    return (per + (K + 2) * U32) * absprod + 1e-30


# ---- 8192-point STFT and iSTFT ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("hop", [1024, 2048, 441])
def test_stft_8192_elementwise(ops, hop):
    N, L = 8192, 3 * 8192 + 517
    wav = torch.randn((2, L), generator=_gen(hop), dtype=torch.float64) * 0.3 + 0.2
    got = ops.stft(wav.float().to(DEV), N, hop).cpu().double()
    xp = np.pad(wav.float().double().numpy(), ((0, 0), (N // 2, N // 2)), mode="reflect")
    T = 1 + L // hop
    assert got.shape == (2, T, N // 2 + 1, 2)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)
    fr = np.stack([xp[:, t * hop:t * hop + N] * win for t in range(T)], 1)          # [2, T, N] float64
    ref = np.fft.rfft(fr, axis=-1)
    err = np.abs(got[..., 0].numpy() - ref.real) + np.abs(got[..., 1].numpy() - ref.imag)
    # radix-4 Stockham in fp32: about log2(N) roundings of twiddled partial sums, each at most the frame's L1 norm
    bound = 4 * (math.log2(N) + 4) * U32 * np.abs(fr).sum(-1, keepdims=True) * 2
    assert (err <= bound).all(), float((err / bound).max())


@pytest.mark.parametrize("hop,S", [(1024, 2), (2048, 1)])
def test_istft_8192_vs_float64(ops, hop, S):
    N, B, T = 8192, 2, 12
    c = torch.randn((B * S, T, N // 2 + 1, 2), generator=_gen(7 + hop), dtype=torch.float64)
    got = ops.istft(c.float().to(DEV), B, S, N, hop).cpu().double()
    cc = torch.view_as_complex(c.float().double().contiguous())
    ref = torch.istft(cc.transpose(1, 2), N, hop, N, torch.hann_window(N, dtype=torch.float64), center=True)
    assert got.shape == ref.shape
    # each output sample is a sum over <= N / hop frames of inverse FFTs of N / 2 + 1 bins, divided by the window envelope
    scale = c.abs().sum((2, 3)).max() / N
    assert float((got - ref).abs().max()) <= 8 * (math.log2(N) + 8) * U32 * float(scale) * (N // hop) * 4


def test_stft_8192_roundtrip(ops):
    wav = torch.randn((2, 261120), generator=_gen(5)).to(DEV) * 0.4
    c = ops.stft(wav, 8192, 1024)
    back = ops.istft(c, 1, 2, 8192, 1024)
    assert float((back - wav).abs().max()) <= 2e-5


# ---- plane instance norm ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C,pitch,c0", [(2, 40, 300, 40, 48, 4), (1, 64, 512, 128, 128, 0), (3, 3, 5, 7, 7, 0)])
def test_instnorm_plane_elementwise(ops, B, H, W, C, pitch, c0):
    g = _gen(B * H + C)
    buf = torch.randn((B, H, W, pitch), generator=g) * 0.5 + 3.0          # DC-heavy: the shifted sums matter
    gamma, beta = 0.5 + torch.rand(C, generator=g), 0.1 * torch.randn(C, generator=g)
    out = torch.full((B, H, W, pitch + 4), 7.0)
    xb, ob = buf.to(DEV), out.to(DEV)
    ops.instnorm_plane(ops.CLView(xb, c0, C), gamma.to(DEV), beta.to(DEV), ops.CLView(ob, 2, C))
    got = ob.cpu().double()
    x = buf[..., c0:c0 + C].double()
    mean = x.mean((1, 2), keepdim=True)
    var = x.var((1, 2), unbiased=False, keepdim=True)
    zz = (x - mean) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()
    ref = 0.5 * zz * (1 + torch.erf(zz / math.sqrt(2)))
    # each statistic is a sum of at most 2048 / 8 per lane, 8 lanes and n / 2048 chunks of shifted values, so its relative
    # error is below (256 + 8 + n / 2048 + 16) u; z = (x - mean) / std then errs by that much relative, times a margin
    # for the shift (|x - shift| / std) and the fp32 normalise and GELU
    n = H * W
    steps = 256 + 8 + n / 2048 + 16
    spread = (x - x[:, :1, :1]).abs().amax((1, 2), keepdim=True) / torch.sqrt(var + 1e-5)
    z = (x - mean) / torch.sqrt(var + 1e-5)
    tol = 4 * steps * U32 * (1 + spread) ** 2 * (1 + z.abs()) * gamma.double() + 16 * U32 * (1 + ref.abs())
    assert ((got[..., 2:2 + C] - ref).abs() <= tol).all(), float(((got[..., 2:2 + C] - ref).abs() / tol).max())
    assert (got[..., :2] == 7.0).all() and (got[..., 2 + C:] == 7.0).all()
    # an item normalised alone gives the same bits
    one = torch.empty((1, H, W, C), device=DEV)
    ops.instnorm_plane(ops.CLView(xb[B - 1:], c0, C), gamma.to(DEV), beta.to(DEV), ops.CLView(one))
    assert torch.equal(one[0].cpu(), ob[B - 1, ..., 2:2 + C].cpu())


# ---- 2x2 stride-2 conv, transposed conv, TDF Linear ------------------------------------------------------------------
@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("B,H,W,C,N", [(2, 16, 64, 32, 48), (1, 8, 12, 6, 5)])
def test_conv2x2_stride2_elementwise(ops, precise, B, H, W, C, N):
    g = _gen(C * N)
    x, w = torch.randn((B, H, W, C), generator=g), torch.randn((N, C, 2, 2), generator=g) / (4 * C) ** 0.5
    y = torch.empty((B, H // 2, W // 2, N), device=DEV)
    with _precise(precise):
        ops.conv2d(ops.CLView(x.to(DEV)), w.permute(0, 2, 3, 1).contiguous().to(DEV), ops.CLView(y), k=2, stride=2)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), stride=2).permute(0, 2, 3, 1)
    absprod = F.conv2d(x.double().abs().permute(0, 3, 1, 2), w.double().abs(), stride=2).permute(0, 2, 3, 1)
    assert ((y.cpu().double() - ref).abs() <= _contraction_bound(absprod, 4 * C, precise)).all()


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("B,H,W,C,N,pitch,c0", [(2, 8, 32, 64, 48, 96, 0), (1, 3, 5, 7, 5, 12, 6)])
def test_convt2x2_elementwise(ops, precise, B, H, W, C, N, pitch, c0):
    g = _gen(C + N)
    x, w = torch.randn((B, H, W, C), generator=g), torch.randn((C, N, 2, 2), generator=g) / C ** 0.5
    out = torch.full((B, 2 * H, 2 * W, pitch), 7.0, device=DEV)
    with _precise(precise):
        ops.convt2x2(ops.CLView(x.to(DEV)), w.permute(2, 3, 1, 0).contiguous().to(DEV), ops.CLView(out, c0, N))
    ref = F.conv_transpose2d(x.double().permute(0, 3, 1, 2), w.double(), stride=2).permute(0, 2, 3, 1)
    absprod = F.conv_transpose2d(x.double().abs().permute(0, 3, 1, 2), w.double().abs(), stride=2).permute(0, 2, 3, 1)
    got = out.cpu().double()
    assert ((got[..., c0:c0 + N] - ref).abs() <= _contraction_bound(absprod, C, precise)).all()
    rest = torch.cat([got[..., :c0], got[..., c0 + N:]], -1)
    assert (rest == 7.0).all()


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("B,H,K,M,C,pitch", [(2, 6, 256, 64, 128, 128), (1, 5, 40, 10, 7, 12), (1, 2, 130, 300, 70, 72)])
def test_tdf_elementwise(ops, precise, B, H, K, M, C, pitch):
    g = _gen(K + M + C)
    xb = torch.randn((B, H, K, pitch), generator=g)
    w = torch.randn((M, K), generator=g) / K ** 0.5
    r = torch.randn((B, H, M, C), generator=g)
    y = r.clone().to(DEV)
    with _precise(precise):
        ops.mdx_tdf(ops.CLView(xb.to(DEV), pitch - C, C), w.to(DEV), ops.CLView(y), res=ops.CLView(y))   # residual in place
    x = xb[..., pitch - C:].double()
    ref = torch.einsum("mk,bhkc->bhmc", w.double(), x) + r.double()
    absprod = torch.einsum("mk,bhkc->bhmc", w.double().abs(), x.abs()) + r.double().abs()
    assert ((y.cpu().double() - ref).abs() <= _contraction_bound(absprod, K + 1, precise)).all()
    y1, y2 = torch.empty((B, H, M, C), device=DEV), torch.empty((1, H, M, C), device=DEV)
    ops.mdx_tdf(ops.CLView(xb.to(DEV), pitch - C, C), w.to(DEV), ops.CLView(y1))
    ops.mdx_tdf(ops.CLView(xb[B - 1:].contiguous().to(DEV), pitch - C, C), w.to(DEV), ops.CLView(y2))
    assert torch.equal(y2[0].cpu(), y1[B - 1].cpu())        # a slab's result does not depend on the batch


# ---- spectral layouts --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,k,F,nt", [(2, 2, 4, 32, 2), (1, 1, 1, 20, 1), (2, 2, 2, 16, 1)])
def test_front_back_layouts(ops, B, S, k, F, nt):
    T, NB = 6, k * F + 9
    cplx = torch.randn((B * S, T, NB, 2), generator=_gen(B + S + k))
    D = 2 * S * k
    buf = torch.full((B, T, F, D + 3), 7.0, device=DEV)
    ops.mdx_front(cplx.to(DEV), B, S, k, F, ops.CLView(buf, 0, D))
    # the reference: [B, S*2, NB, T] (channel s*2 + re/im), first k F bins, cac2cws, transpose to (T, F)
    x = cplx.reshape(B, S, T, NB, 2).permute(0, 1, 4, 3, 2).reshape(B, S * 2, NB, T)[:, :, :k * F]
    x = x.reshape(B, S * 2, k, F, T).reshape(B, S * 2 * k, F, T).permute(0, 3, 2, 1)
    got = buf.cpu()
    assert torch.equal(got[..., :D], x) and (got[..., D:] == 7.0).all()
    y = torch.randn((B, T, F, nt * D), generator=_gen(9))
    spec = ops.mdx_back(ops.CLView(y.to(DEV)), nt, S, k, NB).cpu()
    # the reference: [B, nt*D, F, T] -> cws2cac -> [B, nt, S*2, kF, T] -> zero bins -> rows (b, target, s)
    z = y.permute(0, 3, 2, 1).reshape(B, nt * D // k, k, F, T).reshape(B, nt * D // k, k * F, T)
    z = torch.cat([z, torch.zeros(B, nt * D // k, NB - k * F, T)], 2).reshape(B * nt * S, 2, NB, T).permute(0, 3, 2, 1)
    assert torch.equal(spec, z.contiguous())


# ---- the whole net -------------------------------------------------------------------------------------------------------
def _model(MX, name):
    case = GOLD[name]
    cfg = O.config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    return MX.MDX23C(cfg).to(DEV).load_state_dict(P), cfg, case


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "mono", "default"])
def test_forward_vs_golden(MX, name, precise):
    m, cfg, case = _model(MX, name)
    shape = case["forward_shape"]
    raw = O.make_audio(case["audio_seed"], (shape[0], cfg["audio"]["num_channels"], cfg["audio"]["chunk_size"]))
    with _precise(precise):
        got = m(raw.to(DEV)).cpu()
    assert tuple(got.shape) == tuple(shape)
    e = rel(got[..., ::case["stride"]], case["forward"])
    print(f"forward {name} precise={precise} rel-L2 {e:.3g}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("name", ["small", "mono"])
def test_demix_vs_golden(MX, name, precise):
    from easevoice_trainer_b200 import bs_roformer
    m, cfg, case = _model(MX, name)
    mix = O.make_audio(case["audio_seed"] + 100, (cfg["audio"]["num_channels"], case["demix_len"]))
    with _precise(precise):
        got = bs_roformer.demix_track(m, mix, DEV)
    assert list(got) == list(case["demix"])
    for key, ref in case["demix"].items():
        e = rel(got[key], ref)
        print(f"demix {name} {key} precise={precise} rel-L2 {e:.3g}")
        assert e <= (TOL_NET_PRECISE if precise else TOL_NET), e


def test_chunk_alone_equals_batched_and_reproducible(MX):
    m, cfg, case = _model(MX, "small")
    raw = O.make_audio(5, (3, 2, cfg["audio"]["chunk_size"])).to(DEV)
    a = m(raw)
    b = m(raw)
    one = m(raw[1:2])
    assert torch.equal(a, b)
    assert torch.equal(one[0], a[1])


def test_forward_input_errors(MX):
    m, cfg, _ = _model(MX, "small")
    for bad in (torch.zeros(1, 2, 7680), torch.zeros(1, 1, 7680, device=DEV), torch.zeros(2, 7680, device=DEV),
                torch.zeros(1, 2, 7680 + 512, device=DEV)):
        with pytest.raises(ValueError):
            m(bad)
