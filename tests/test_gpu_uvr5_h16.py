"""GPU tests of the 16-bit compute type of the UVR5 VR, DeEcho / DeReverb and MDX23C nets (`pytest -m gpu`):
evk_conv2d_fwd_h16 element for element on exactly representable operands and within a float64 rounding bound on random
ones, its batch independence, the nets against the float64 emulation (tests/uvr5_h16_ref.py) and the fp32 goldens, and
switching between compute types."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mdx23c_oracle as MO
from oracle import uvr5_echo_oracle as EO
from oracle import uvr5_oracle as VO
from tests import uvr5_h16_ref as R
from tests.exact_ref import ints

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_VR = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_vr.pt"), weights_only=False)
GOLD_ECHO = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_deecho.pt"), weights_only=False)
GOLD_MDX = torch.load(os.path.join(ROOT, "tests", "golden", "mdx23c.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
H16 = [torch.float16, torch.bfloat16]
U32 = 2.0 ** -24
# rel-L2 of the whole net against the float64 emulation of its compute type, and against the fp32 goldens.  Measured on an
# H100: VR and DeEcho / DeReverb predict / inference at most 1.3e-4 (fp16) and 1.0e-3 (bf16) against the emulation, 1.9e-4
# and 2.2e-3 against the goldens; MDX23C forward / demix_track at most 8.4e-4 and 5.8e-3 against the emulation, 1.5e-3 and
# 1.3e-2 against the goldens.
TOL_EMU = {"vr": {torch.float16: 5e-4, torch.bfloat16: 4e-3}, "mdx": {torch.float16: 2e-3, torch.bfloat16: 1.5e-2}}
TOL_GOLD = {"vr": {torch.float16: 1e-3, torch.bfloat16: 6e-3}, "mdx": {torch.float16: 4e-3, torch.bfloat16: 3e-2}}
ACTS = (0, 1, 2, 3, 4)         # none, relu, lrelu, sigmoid, gelu


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


class _precise:
    def __enter__(self):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(1)

    def __exit__(self, *exc):
        from easevoice_trainer_b200 import lib
        lib.init().evk_set_precise(0)


def rel(a, b):
    a, b = [(t if torch.is_tensor(t) else torch.from_numpy(np.asarray(t))).double().cpu() for t in (a, b)]
    return float((a - b).norm() / b.norm())


# ---- the kernel --------------------------------------------------------------------------------------------------------
# B, H, W, C, N, k, stride, (pad_h, pad_w), (dil_h, dil_w), (extra input channels, input offset), (output offset, extra)
GRID = [
    (2, 16, 20, 2, 16, 3, 1, (1, 1), (1, 1), (0, 0), (0, 0)),          # the first layer: C = 2
    (2, 16, 20, 2, 16, 3, 1, (1, 1), (1, 1), (1, 0), (2, 30)),         # ... from the first two channels of [x | aux]
    (1, 12, 16, 18, 8, 1, 1, (0, 0), (1, 1), (16, 0), (0, 0)),         # bridges: C = 18, 34, 66, 130
    (2, 9, 14, 34, 16, 1, 1, (0, 0), (1, 1), (32, 0), (0, 0)),
    (1, 8, 16, 66, 32, 1, 1, (0, 0), (1, 1), (0, 0), (0, 0)),
    (1, 10, 12, 130, 64, 1, 1, (0, 0), (1, 1), (0, 0), (0, 0)),
    (1, 10, 12, 64, 64, 3, 2, (1, 1), (1, 1), (0, 0), (0, 0)),         # stride 2
    (2, 11, 13, 24, 40, 3, 2, (1, 1), (1, 1), (5, 3), (1, 6)),         # stride 2 from and into odd channel offsets
    (1, 21, 32, 32, 32, 3, 1, (4, 2), (4, 2), (0, 0), (32, 96)),       # DeEcho's ASPP dilations into their concat slice
    (1, 21, 32, 32, 32, 3, 1, (8, 4), (8, 4), (0, 0), (64, 64)),
    (1, 21, 32, 32, 32, 3, 1, (12, 6), (12, 6), (0, 0), (96, 32)),
    (1, 5, 3, 16, 24, 3, 1, (12, 6), (12, 6), (0, 0), (0, 0)),         # every tap but the centre in the padding
    (2, 16, 16, 16, 24, 2, 2, (0, 0), (1, 1), (0, 0), (0, 0)),         # MDX23C's 2x2 stride-2 downscale
    (1, 9, 7, 12, 20, 3, 1, (2, 0), (1, 1), (1, 1), (3, 1)),           # per-axis padding
    (1, 9, 7, 12, 20, 3, 1, (0, 3), (2, 6), (0, 0), (0, 0)),
    (2, 8, 8, 7, 1, 3, 1, (1, 1), (1, 1), (2, 1), (0, 2)),             # N = 1 (the LSTM module's 1x1 has C = 2 ch)
    (1, 8, 8, 20, 5, 1, 1, (0, 0), (1, 1), (0, 0), (0, 0)),
    (1, 8, 12, 40, 33, 3, 1, (1, 1), (1, 1), (0, 0), (0, 0)),          # N just past a column tile
    (1, 8, 12, 48, 100, 3, 1, (1, 1), (1, 1), (0, 0), (0, 0)),
    (1, 6, 8, 136, 200, 3, 1, (1, 1), (1, 1), (0, 0), (0, 0)),         # two column tiles of 128
    (1, 6, 8, 45, 300, 1, 1, (0, 0), (1, 1), (3, 1), (1, 2)),          # three, with odd input and output offsets
]


def _case_operands(case, gen, make_x, make_w):
    B, H, W, C, N, k, s, (ph, pw), (dh, dw), (xe, xo), (yo, ye) = case
    xbuf = torch.full((B, H, W, C + xe), float("nan"))        # channels outside the slice must not be read
    xbuf[..., xo:xo + C] = make_x((B, H, W, C))
    w = make_w((N, k, k, C))
    Ho, Wo = (H + 2 * ph - dh * (k - 1) - 1) // s + 1, (W + 2 * pw - dw * (k - 1) - 1) // s + 1
    return xbuf, w, (Ho, Wo)


def _run(ops, case, xbuf, w, dtype, act, scale, bias, fp32=False):
    B, H, W, C, N, k, s, pad, dil, (xe, xo), (yo, ye) = case
    Ho, Wo = (H + 2 * pad[0] - dil[0] * (k - 1) - 1) // s + 1, (W + 2 * pad[1] - dil[1] * (k - 1) - 1) // s + 1
    ybuf = torch.full((B, Ho, Wo, yo + N + ye), 7.0, device=DEV)
    x = ops.CLView(xbuf.to(DEV), xo, C)
    kw = dict(k=k, stride=s, pad=pad, dil=dil, scale=scale.to(DEV), bias=bias.to(DEV), act=act)
    if fp32:
        ops.conv2d(x, w.float().contiguous().to(DEV), ops.CLView(ybuf, yo, N), **kw)
    else:
        ops.conv2d_h16(x, ops.pack_conv_h16(w.float().to(DEV), dtype), ops.CLView(ybuf, yo, N), **kw)
    y = ybuf.cpu()
    assert (y[..., :yo] == 7).all() and (y[..., yo + N:] == 7).all()       # nothing outside the slice is written
    return y[..., yo:yo + N]


def _ref(case, x, w):
    """float64 conv of channels-last x [B, H, W, C] (the slice) and w [N, k, k, C] -> [B, Ho, Wo, N]"""
    B, H, W, C, N, k, s, pad, dil, _, _ = case
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), None, s, pad, dil).permute(0, 2, 3, 1)


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("case", GRID)
def test_conv2d_h16_exact(ops, case, dtype):
    """Small integers are exact in fp16 and bf16 and every partial sum is an exact fp32 integer, so the kernel must give the
    float64 result bit for bit; with a power-of-two scale and a bias on a 1/4 grid the epilogue is exact too, and for every
    activation the kernel equals the TF32 kernel, whose epilogue it shares, on the same exact operands."""
    g = torch.Generator().manual_seed(hash(case) % 10007)
    xbuf, w, _ = _case_operands(case, g, lambda s: ints(s, 3, g).float(), lambda s: ints(s, 2, g))
    N, xo, C = case[4], case[9][1], case[3]
    scale = 2.0 ** torch.randint(-2, 2, (N,), generator=g).float()
    bias = ints((N,), 8, g).float() / 4
    ref = _ref(case, xbuf[..., xo:xo + C], w) * scale.double() + bias.double()
    for act in ACTS:
        got = _run(ops, case, xbuf, w, dtype, act, scale, bias)
        if act == 0:
            assert torch.equal(got.double(), ref)
        elif act == 1:
            assert torch.equal(got.double(), ref.clamp(min=0))
        assert torch.equal(got, _run(ops, case, xbuf, w, dtype, act, scale, bias, fp32=True)), act


def _trunc(t, dtype):
    """fp32 t with its mantissa cut to dtype's (round toward zero; normal fp16 range)"""
    return (t.float().view(torch.int32) & (~0x1FFF if dtype == torch.float16 else ~0xFFFF)).view(torch.float32)


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("case,positive", [(GRID[i], j % 2 == 0) for j, i in enumerate((0, 3, 6, 7, 8, 12, 14, 19, 20))])
def test_conv2d_h16_rounding_bound(ops, case, positive, dtype):
    """Random operands: |y - h(x) * h(w)| within the fp32 accumulation bound 2 K u32 sum |h(x) h(w)| plus the epilogue's
    rounding, element by element.  With positive operands, whose truncation errors add up instead of cancelling, the same
    bound fails for operands truncated instead of rounded."""
    g = torch.Generator().manual_seed(hash(case) % 10007 + 1)
    sign = (lambda t: t.abs()) if positive else (lambda t: t)
    xbuf, w, _ = _case_operands(case, g, lambda s: sign(torch.randn(s, generator=g)),
                                lambda s: sign(torch.randn(s, generator=g)) / (s[1] * s[2] * s[3]) ** 0.5)
    N, xo, C, k = case[4], case[9][1], case[3], case[5]
    scale, bias = 0.5 + torch.rand(N, generator=g), 0.1 * torch.randn(N, generator=g)
    x = xbuf[..., xo:xo + C]
    h = R.rounding(dtype)
    acc = _ref(case, h(x), h(w))
    ref = acc * scale.double() + bias.double()
    K = k * k * C
    bound = (2 * K * U32 * _ref(case, h(x).abs(), h(w).abs()) * scale.double() + 2 * U32 * (acc.abs() * scale.double()
             + bias.double().abs()) + 1e-30)
    got = _run(ops, case, xbuf, w, dtype, 0, scale, bias).double()
    worst = float(((got - ref).abs() / bound).max())
    print(f"{case} {dtype}: largest error {worst:.3f} of the bound")
    assert worst <= 1.0
    if positive:
        trunc = _ref(case, _trunc(x, dtype), _trunc(w, dtype)) * scale.double() + bias.double()
        assert ((trunc - ref).abs() > bound).any()


@pytest.mark.parametrize("dtype", H16)
def test_conv2d_h16_batch_independent(ops, dtype):
    g = torch.Generator().manual_seed(5)
    B, H, W, C, N = 16, 21, 32, 34, 40
    x = torch.randn(B, H, W, C + 2, generator=g).to(DEV)
    w = ops.pack_conv_h16(torch.randn(N, 3, 3, C, generator=g).to(DEV) / 17, dtype)
    kw = dict(k=3, pad=(4, 2), dil=(4, 2), act=2)
    y = torch.empty(B, H, W, N, device=DEV)
    ops.conv2d_h16(ops.CLView(x, 1, C), w, ops.CLView(y), **kw)
    with _precise():                                   # evk_set_precise has no effect on the 16-bit kernel
        for b in (0, 5, 15):
            one = torch.empty(1, H, W, N, device=DEV)
            ops.conv2d_h16(ops.CLView(x[b:b + 1].contiguous(), 1, C), w, ops.CLView(one), **kw)
            assert torch.equal(one[0], y[b])


def test_conv2d_h16_rejects_bad_packs(ops):
    x = torch.zeros(1, 4, 4, 8, device=DEV)
    y = torch.zeros(1, 4, 4, 4, device=DEV)
    w = ops.pack_conv_h16(torch.zeros(4, 3, 3, 8, device=DEV), torch.float16)
    with pytest.raises(AssertionError):                        # K of a different C
        ops.conv2d_h16(ops.CLView(x, 0, 4), w, ops.CLView(y), k=3, pad=1)
    with pytest.raises(RuntimeError, match="packed weight pitch"):
        bad = ops.PackedH16(w.w[:, :48].contiguous(), 72)
        ops.conv2d_h16(ops.CLView(x), bad, ops.CLView(y), k=3, pad=1)


# ---- the nets ----------------------------------------------------------------------------------------------------------
def _vr_net(case):
    from easevoice_trainer_b200 import uvr5
    g = GOLD_VR[case]
    P = VO.init_params(VO.param_spec(g["size"]), g["seed"])
    return uvr5.get_nets_model(g["n_fft"], g["size"]).to(DEV).load_state_dict(P), P, g


def _echo_net(case):
    from easevoice_trainer_b200 import uvr5
    g = GOLD_ECHO[case]
    P = EO.init_params(EO.param_spec(g["n_fft"], g["nout"]), g["seed"])
    return uvr5.CascadedNet(g["n_fft"], g["nout"]).to(DEV).load_state_dict(P), P, g


def _predict_input(g, n=None):
    bins = g["n_fft"] // 2 + 1
    n = n or g["predict_windows"]
    x = torch.from_numpy(np.abs(VO.make_spec(g["spec_seed"] + 100, bins, 512 * n)))
    x = x.reshape(2, bins, n, 512).permute(2, 0, 1, 3).contiguous()
    return (x / x.max()).to(DEV)


def _vr_agg(g):
    return {"value": g["agg"] / 100, "split_bin": g["split_bin"], "aggr_correction": None}


@pytest.mark.parametrize("dtype", H16)
def test_vr_predict_vs_emulation(ops, dtype):
    net, P, g = _vr_net("small")
    x = _predict_input(g)
    got = net.set_compute_type(dtype).predict(x, _vr_agg(g))
    enlarge = VO.SIZES[g["size"]]["enlarge"]
    e = rel(got, R.vr_predict(P, x, _vr_agg(g), dtype, g["n_fft"], enlarge))
    eg = rel(got[..., ::g["stride"]], g["predict_out"])
    print(f"vr predict small {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
    assert e <= TOL_EMU["vr"][dtype] and eg <= TOL_GOLD["vr"][dtype]
    assert torch.equal(net.forward(x, _vr_agg(g))[..., 128:-128], got)


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("case", ["small", "full"])
def test_vr_inference_vs_emulation(ops, case, dtype):
    from easevoice_trainer_b200 import uvr5
    net, P, g = _vr_net(case)
    net.set_compute_type(dtype)
    spec = VO.make_spec(g["spec_seed"], g["n_fft"] // 2 + 1, g["n_frame"])
    data = {"window_size": 512, "tta": g["tta"]}
    pred = uvr5.inference(spec, DEV, net, _vr_agg(g), data)[0]
    enlarge = VO.SIZES[g["size"]]["enlarge"]
    emu = R.inference(lambda w: R.vr_predict(P, w, _vr_agg(g), dtype, g["n_fft"], enlarge), spec, data, VO.OFFSET, DEV)
    e, eg = rel(pred, emu), rel(pred[..., ::g["stride"]], g["pred"])
    print(f"vr inference {case} {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
    assert e <= TOL_EMU["vr"][dtype] and eg <= TOL_GOLD["vr"][dtype]


@pytest.mark.parametrize("dtype", H16)
def test_echo_predict_vs_emulation(ops, dtype):
    net, P, g = _echo_net("small")
    x = _predict_input(g)
    got = net.set_compute_type(dtype).predict(x)
    e = rel(got, R.echo_predict(P, x, dtype, g["n_fft"]))
    eg = rel(got[..., ::g["stride"]], g["predict_out"])
    print(f"echo predict small {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
    assert e <= TOL_EMU["vr"][dtype] and eg <= TOL_GOLD["vr"][dtype]
    assert torch.equal((x * net.forward(x))[..., 64:-64], got)


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("case", ["small", "deecho", "dereverb"])
def test_echo_inference_vs_emulation(ops, case, dtype):
    from easevoice_trainer_b200 import uvr5
    net, P, g = _echo_net(case)
    net.set_compute_type(dtype)
    spec = EO.make_spec(g["spec_seed"], g["n_fft"] // 2 + 1, g["n_frame"])
    data = {"window_size": 512, "tta": g["tta"]}
    agg = {"value": g["agg"] / 100, "split_bin": 85, "aggr_correction": None}
    pred = uvr5.inference(spec, DEV, net, agg, data)[0]
    lstms = EO.lstm_modules({k: (v.double() if v.is_floating_point() else v) for k, v in P.items()}, DEV, torch.float64)
    emu = R.inference(lambda w: R.echo_predict(P, w, dtype, g["n_fft"], lstms), spec, data, EO.OFFSET, DEV)
    e, eg = rel(pred, emu), rel(pred[..., ::g["stride"]], g["pred"])
    print(f"echo inference {case} {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
    assert e <= TOL_EMU["vr"][dtype] and eg <= TOL_GOLD["vr"][dtype]


def _mdx(name):
    from easevoice_trainer_b200 import mdx23c
    case = GOLD_MDX[name]
    cfg = MO.config(case["over"])
    P = MO.init_params(MO.param_spec(cfg), case["seed"])
    return mdx23c.MDX23C(cfg).to(DEV).load_state_dict(P), P, cfg, case


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("name", ["small", "mono", "default"])
def test_mdx_forward_vs_emulation(ops, name, dtype):
    m, P, cfg, case = _mdx(name)
    shape = case["forward_shape"]
    raw = MO.make_audio(case["audio_seed"], (shape[0], cfg["audio"]["num_channels"], cfg["audio"]["chunk_size"])).to(DEV)
    got = m.set_compute_type(dtype)(raw)
    emu = R.mdx_forward(P, cfg, raw, dtype)
    if name == "default" and dtype == torch.float16:
        # the 8K-FFT configuration's final_conv input leaves fp16's range: h(x) is +-inf there, in the kernel as in a
        # torch cast, so the output is not finite -- in the emulation too
        assert not torch.isfinite(got).all() and not torch.isfinite(emu).all()
        return
    assert torch.isfinite(got).all()
    e, eg = rel(got, emu), rel(got.cpu()[..., ::case["stride"]], case["forward"])
    print(f"mdx23c forward {name} {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
    assert e <= TOL_EMU["mdx"][dtype] and eg <= TOL_GOLD["mdx"][dtype]


@pytest.mark.parametrize("dtype", H16)
@pytest.mark.parametrize("name", ["small", "mono"])
def test_mdx_demix_vs_emulation(ops, name, dtype):
    from easevoice_trainer_b200 import bs_roformer
    m, P, cfg, case = _mdx(name)
    mix = MO.make_audio(case["audio_seed"] + 100, (cfg["audio"]["num_channels"], case["demix_len"]))
    got = bs_roformer.demix_track(m.set_compute_type(dtype), mix, DEV)
    emu = R.mdx_demix(P, cfg, mix, dtype, DEV)
    assert list(got) == list(emu) == list(case["demix"])
    for key in got:
        e, eg = rel(got[key], emu[key]), rel(got[key], case["demix"][key])
        print(f"mdx23c demix {name} {key} {dtype}: rel-L2 {e:.3e} against the emulation, {eg:.3e} against the fp32 golden")
        assert e <= TOL_EMU["mdx"][dtype] and eg <= TOL_GOLD["mdx"][dtype]


# ---- switching ---------------------------------------------------------------------------------------------------------
def _batch_and_alone(run, x):
    a = run(x)
    for i in (0, x.shape[0] - 1):
        assert torch.equal(run(x[i:i + 1]), a[i:i + 1])
    return a


@pytest.mark.parametrize("which", ["vr", "echo", "mdx"])
def test_switching_and_precise_mode(ops, which):
    if which == "mdx":
        m, _, cfg, _ = _mdx("small")
        fresh = _mdx("small")[0]
        x = MO.make_audio(9, (3, 2, cfg["audio"]["chunk_size"])).to(DEV)
        run = m
    else:
        m, _, g = (_vr_net if which == "vr" else _echo_net)("small")
        fresh = (_vr_net if which == "vr" else _echo_net)("small")[0]
        x = torch.cat([_predict_input(g), _predict_input(g).flip(-1)], 0)
        run = m.predict
    ref32 = fresh.predict(x) if which != "mdx" else fresh(x)
    out = {}
    for dt in (torch.float16, None, torch.bfloat16, torch.float16, None, torch.bfloat16):
        m.set_compute_type(dt)
        y = _batch_and_alone(run, x)
        if dt is None:
            assert torch.equal(y, ref32)                         # the bits of a fresh fp32 model
        else:
            if dt in out:
                assert torch.equal(y, out[dt])
            out[dt] = y
            if which != "mdx":      # MDX23C's TDF Linears and transposed convs stay fp32 and follow evk_set_precise
                with _precise():
                    assert torch.equal(run(x), y)               # the precise mode does not touch the 16-bit path
    assert not torch.equal(out[torch.float16], ref32) and not torch.equal(out[torch.bfloat16], out[torch.float16])
