"""GPU tests of the UVR5 DeEcho / DeReverb separator (`pytest -m gpu`): the anisotropic 2-D convolution
(evk_conv2d_fwd) and the bidirectional LSTM recurrence (evk_lstm_bidir_fwd) against float64, their reproducibility and
batch independence, and CascadedNet.predict / uvr5.inference against the outputs the reference computed
(tests/golden/uvr5_deecho.pt, pinned by oracle/pin_uvr5_echo.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import uvr5_echo_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_deecho.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
# rel-L2 of the whole net against the fp32 reference.  Measured on an H100: TF32 1.3e-4 (small, predict and inference),
# 1.3e-4 (deecho) and 1.8e-4 (dereverb); 3xTF32 1.2e-6 to 1.3e-6 (small), 2.1e-6 (deecho) and 2.4e-6 (dereverb).  The
# LSTM's two projection GEMMs stay TF32 under 3xTF32, which sets the floor of the precise figures.
TOL_NET, TOL_NET_PRECISE = 1e-3, 1e-5


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


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
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---- anisotropic convolution ------------------------------------------------------------------------------------------
# B, H, W, C, N, k, stride, (dil_h, dil_w), act, (extra input channels, input channel offset), (output offset, extra)
CONV_HW_GRID = [
    (2, 21, 32, 96, 96, 3, 1, (4, 2), 1, (0, 0), (96, 288)),        # the band nets' ASPP branches into their concat slice
    (2, 21, 32, 96, 96, 3, 1, (8, 4), 1, (0, 0), (192, 192)),
    (2, 21, 32, 96, 96, 3, 1, (12, 6), 1, (0, 0), (288, 96)),
    (1, 42, 32, 128, 128, 3, 1, (4, 2), 1, (0, 0), (0, 0)),         # the full-band net's ASPP
    (1, 42, 32, 128, 128, 3, 1, (8, 4), 1, (0, 0), (0, 0)),
    (1, 42, 32, 128, 64, 3, 1, (12, 6), 1, (8, 4), (4, 8)),         # channel-sliced input and output
    (1, 5, 3, 16, 24, 3, 1, (12, 6), 0, (0, 0), (0, 0)),            # every tap but the centre in the padding
    (2, 13, 4, 20, 8, 3, 1, (8, 4), 2, (3, 1), (5, 3)),             # unaligned slice: the mma.sync path
    (1, 21, 32, 24, 40, 3, 2, (4, 2), 2, (4, 4), (0, 0)),           # stride 2
    (3, 9, 7, 12, 20, 3, 1, (2, 6), 1, (0, 0), (3, 1)),             # columns dilated more than rows
]


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("case", CONV_HW_GRID)
def test_conv2d_hw_vs_float64(ops, case, precise):
    B, H, W, C, N, k, s, (dh, dw), act, (xe, xo), (yo, ye) = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    xbuf = torch.randn(B, H, W, C + xe, generator=g).to(DEV)
    w = (torch.randn(N, C, k, k, generator=g) / (C * k * k) ** 0.5).double()
    scale, bias = 0.5 + torch.rand(N, generator=g), 0.1 * torch.randn(N, generator=g)
    pad = (dh * (k // 2), dw * (k // 2))
    Ho, Wo = ops.conv2d_out(H, k, s, pad[0], dh), ops.conv2d_out(W, k, s, pad[1], dw)
    ybuf = torch.full((B, Ho, Wo, yo + N + ye), 7.0, device=DEV)
    with _precise(precise):
        ops.conv2d(ops.CLView(xbuf, xo, C), w.float().permute(0, 2, 3, 1).contiguous().to(DEV), ops.CLView(ybuf, yo, N),
                   k=k, stride=s, pad=pad, dil=(dh, dw), scale=scale.to(DEV), bias=bias.to(DEV), act=act)
    x64 = xbuf[..., xo:xo + C].double().cpu().permute(0, 3, 1, 2)
    ref = F.conv2d(x64, w, None, s, pad, (dh, dw)) * scale.double()[:, None, None] + bias.double()[:, None, None]
    ref = [lambda t: t, F.relu, lambda t: F.leaky_relu(t, 0.01), torch.sigmoid][act](ref).permute(0, 2, 3, 1)
    got = ybuf.cpu()
    e = rel(got[..., yo:yo + N], ref)
    assert e <= (5e-6 if precise else 2e-3), e
    assert (got[..., :yo] == 7).all() and (got[..., yo + N:] == 7).all()       # nothing outside the slice is written


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("case", [(2, 21, 32, 64, 48, 3, 1, 4, 1), (1, 17, 9, 20, 40, 3, 2, 1, 2), (2, 8, 8, 6, 5, 1, 1, 1, 0)])
def test_conv2d_hw_equal_axes_bit_identical(ops, case, precise):
    B, H, W, C, N, k, s, d, act = case
    x = torch.randn(B, H, W, C, device=DEV)
    w = torch.randn(N, k, k, C, device=DEV) / (C * k * k) ** 0.5
    scale, bias = 0.5 + torch.rand(N, device=DEV), 0.1 * torch.randn(N, device=DEV)
    p = d * (k // 2)
    Ho, Wo = ops.conv2d_out(H, k, s, p, d), ops.conv2d_out(W, k, s, p, d)
    a, b = torch.empty(B, Ho, Wo, N, device=DEV), torch.empty(B, Ho, Wo, N, device=DEV)
    with _precise(precise):
        ops.conv2d(ops.CLView(x), w, ops.CLView(a), k=k, stride=s, pad=p, dil=d, scale=scale, bias=bias, act=act)
        ops.conv2d(ops.CLView(x), w, ops.CLView(b), k=k, stride=s, pad=(p, p), dil=(d, d), scale=scale, bias=bias, act=act)
    assert torch.equal(a, b)


# ---- LSTM recurrence --------------------------------------------------------------------------------------------------
def _lstm_case(H, I, T, N, seed):
    """-> (G fp32 [T, N, 8H] on the device, w_hh [2, 4H, H] on the device, float64 nn.LSTM output [T, N, 2H])"""
    g = torch.Generator().manual_seed(seed)
    m = torch.nn.LSTM(I, H, bidirectional=True).double()
    with torch.no_grad():
        for prm in m.parameters():
            prm.copy_((torch.rand(prm.shape, generator=g, dtype=torch.float64) * 2 - 1) / H ** 0.5)
    x = torch.randn(T, N, I, generator=g, dtype=torch.float64)
    with torch.no_grad():
        ref = m(x)[0]
    G = torch.cat([x @ getattr(m, "weight_ih_l0" + s).t() + getattr(m, "bias_ih_l0" + s) + getattr(m, "bias_hh_l0" + s)
                   for s in ("", "_reverse")], -1)
    w_hh = torch.stack([m.weight_hh_l0, m.weight_hh_l0_reverse])
    return G.float().to(DEV).contiguous(), w_hh.float().to(DEV).contiguous(), ref


@pytest.mark.parametrize("T", [1, 7, 256])
@pytest.mark.parametrize("I", [16, 168, 336])
@pytest.mark.parametrize("H", [32, 64])
def test_lstm_vs_float64(ops, H, I, T):
    for N in (1, 3, 16, 33):
        G, w_hh, ref = _lstm_case(H, I, T, N, seed=H * 7 + I + T * 3 + N)
        y = ops.lstm_bidir(G, w_hh)
        e = rel(y, ref)
        assert y.shape == (T, N, 2 * H) and e <= 2e-6, (N, e)
        # the same rows in (n, t) order
        y2 = ops.lstm_bidir(G.transpose(0, 1).contiguous(), w_hh, order="nt")
        assert torch.equal(y2.transpose(0, 1), y)


def test_lstm_rejects_unsupported_hidden(ops):
    for H in (16, 48, 128):
        G = torch.zeros(4, 2, 8 * H, device=DEV)
        with pytest.raises(RuntimeError, match=f"hidden size {H}"):
            ops.lstm_bidir(G, torch.zeros(2, 4 * H, H, device=DEV))


def test_lstm_reproducible_and_batch_independent(ops):
    G, w_hh, _ = _lstm_case(64, 336, 256, 140, seed=11)         # 140 rows: two rows per CTA
    a = ops.lstm_bidir(G, w_hh)
    assert torch.equal(a, ops.lstm_bidir(G, w_hh))
    for n in (0, 1, 77, 139):
        assert torch.equal(ops.lstm_bidir(G[:, n:n + 1].contiguous(), w_hh), a[:, n:n + 1])
    assert torch.equal(ops.lstm_bidir(G[:, 5:21].contiguous(), w_hh), a[:, 5:21])


# ---- the whole net ----------------------------------------------------------------------------------------------------
def _params(case, fp16=False):
    g = GOLD[case]
    P = O.init_params(O.param_spec(g["n_fft"], g["nout"]), g["seed"])
    return {k: (v.half() if v.is_floating_point() else v) for k, v in P.items()} if fp16 else P


def _net(case, fp16=False):
    from easevoice_trainer_b200 import uvr5
    g = GOLD[case]
    return uvr5.CascadedNet(g["n_fft"], g["nout"]).to(DEV).load_state_dict(_params(case, fp16))


def _agg(g):
    return {"value": g["agg"] / 100, "split_bin": 85, "aggr_correction": None}


def _predict_input(g):
    bins = g["n_fft"] // 2 + 1
    x = torch.from_numpy(np.abs(O.make_spec(g["spec_seed"] + 100, bins, 512 * g["predict_windows"])))
    x = x.reshape(2, bins, g["predict_windows"], 512).permute(2, 0, 1, 3).contiguous()
    return (x / x.max()).to(DEV)


@pytest.mark.parametrize("precise", [False, True])
def test_predict_golden(ops, precise):
    g = GOLD["small"]
    net = _net("small")
    with _precise(precise):
        out = net.predict(_predict_input(g), _agg(g))
    e = rel(out[..., ::g["stride"]], g["predict_out"])
    print(f"predict small precise={precise}: rel-L2 {e:.3e}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET)


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("case", ["small", "deecho", "dereverb"])
def test_inference_golden(ops, case, precise):
    from easevoice_trainer_b200 import uvr5
    g = GOLD[case]
    net = _net(case)
    spec = O.make_spec(g["spec_seed"], g["n_fft"] // 2 + 1, g["n_frame"])
    with _precise(precise):
        pred, mag, phase = uvr5.inference(spec, DEV, net, _agg(g), {"window_size": 512, "tta": g["tta"]})
    assert pred.dtype == np.float32 and pred.shape == (2, g["n_fft"] // 2 + 1, g["n_frame"])
    pred = pred[..., ::g["stride"]]                      # the golden keeps every stride-th frame
    assert np.array_equal(mag, np.abs(spec)) and np.array_equal(phase, np.exp(1.0j * np.angle(spec)))
    e = rel(torch.from_numpy(pred), g["pred"])
    print(f"inference {case} precise={precise}: rel-L2 {e:.3e}")
    assert e <= (TOL_NET_PRECISE if precise else TOL_NET)


def test_reproducible_batch_independent_and_forward(ops):
    g = GOLD["small"]
    net = _net("small")
    x = torch.cat([_predict_input(g), _predict_input(g).flip(-1)], 0)         # 4 windows
    a = net.predict(x)
    assert torch.equal(a, net.predict(x))
    assert torch.equal(a, net.predict(x, {"value": 0.9, "split_bin": 3, "aggr_correction": None}))   # ignored
    for i in range(x.shape[0]):
        assert torch.equal(net.predict(x[i:i + 1]), a[i:i + 1])
    m = net.forward(x)                                   # the mask, as nets_new.CascadedNet.forward returns
    assert m.shape == x.shape and torch.equal((x * m)[..., 64:-64], a)


def test_max_windows_chunking(ops):
    from easevoice_trainer_b200 import uvr5
    g = GOLD["small"]
    net = _net("small")
    spec = O.make_spec(5, 65, 900)
    data = {"window_size": 512, "tta": True}
    ref = uvr5.inference(spec, DEV, net, None, data)[0]
    for mw in (1, 3):
        assert np.array_equal(uvr5.inference(spec, DEV, net, None, data, max_windows=mw)[0], ref)


def test_from_pretrained_fp16(ops, tmp_path):
    from easevoice_trainer_b200 import uvr5
    g = GOLD["small"]
    path = tmp_path / "VR-DeEchoNormal.pth"
    torch.save(_params("small", fp16=True), path)
    net = uvr5.CascadedNet.from_pretrained(str(path), n_fft=g["n_fft"])
    assert (net.nout, net.nout_lstm) == (16, 128)
    x = _predict_input(g)
    assert torch.equal(net.predict(x), _net("small", fp16=True).predict(x))
    with _precise():
        e = rel(net.predict(x)[..., ::g["stride"]], g["predict_out"])
    print(f"fp16 weights: rel-L2 {e:.3e}")
    assert e <= 1e-2


def test_zero_input_is_nan_like_the_reference(ops):
    from easevoice_trainer_b200 import uvr5
    net = _net("small")
    with np.errstate(invalid="ignore"):
        pred, mag, phase = uvr5.inference(np.zeros((2, 65, 40), np.complex64), DEV, net, None,
                                          {"window_size": 512, "tta": False})
    assert pred.shape == (2, 65, 40) and np.isnan(pred).all()
    assert not mag.any() and np.array_equal(phase, np.ones_like(phase))
