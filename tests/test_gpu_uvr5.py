"""GPU tests of the UVR5 VR separator (`pytest -m gpu`): the 2-D convolution family (evk_conv2d_fwd, depthwise, bilinear
resize, height mean, mask head) against float64, bit-reproducibility, batch independence, and CascadedASPPNet.predict /
uvr5.inference against the outputs the reference computed (tests/golden/uvr5_vr.pt, pinned by oracle/pin_uvr5.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import uvr5_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_vr.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
# rel-L2 of the whole net against the fp32 reference.  Measured on an H100: TF32 6.6e-5 (small) and 1.9e-4 (full, four
# cascaded U-nets at 673 bins); 3xTF32 1.3e-7 and 3.6e-7.
TOL_NET, TOL_NET_PRECISE = 1e-3, 2e-6


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


def _act64(v, act):
    return [lambda t: t, F.relu, lambda t: F.leaky_relu(t, 0.01), torch.sigmoid][act](v)


# B, H, W, C, N, k, stride, dil, act, extra input channels (pitch) / input channel offset, output channel offset / extra
CONV_GRID = [
    (1, 16, 32, 2, 16, 3, 1, 1, 2, (0, 0), (0, 0)),            # first layer: C = 2
    (2, 21, 32, 256, 256, 1, 1, 1, 1, (0, 0), (256, 1024)),    # ASPP 1x1 into its concat slice
    (1, 42, 64, 768, 128, 3, 1, 1, 1, (0, 0), (0, 0)),         # decoder, 768 input channels
    (2, 17, 9, 24, 40, 3, 2, 1, 2, (8, 3), (5, 7)),            # odd sizes, stride 2, offsets and pitches on both sides
    (1, 7, 5, 33, 2, 3, 2, 1, 3, (0, 0), (0, 0)),              # tiny odd image, N = 2, sigmoid
    (1, 21, 32, 64, 64, 3, 1, 4, 1, (0, 0), (0, 0)),           # dilation 4
    (1, 21, 32, 64, 48, 3, 1, 16, 0, (16, 16), (0, 16)),       # dilation 16: most taps in the padding
    (3, 1, 31, 96, 768, 1, 1, 1, 1, (0, 0), (0, 0)),           # one row (the pooled ASPP branch), N = 768
    (1, 2, 2, 5, 3, 3, 2, 4, 0, (3, 1), (0, 2)),               # 2 x 2 input, everything padding but the centre
    (1, 3, 3, 768, 2, 1, 2, 1, 0, (0, 0), (0, 0)),             # 1x1 stride 2
    (2, 17, 9, 24, 40, 3, 2, 1, 2, (8, 4), (5, 7)),            # as above with 16-byte-aligned input slices
    (3, 11, 13, 12, 20, 3, 1, 1, 1, (4, 4), (3, 0)),           # N = 20, odd output offset
    (2, 40, 72, 64, 136, 3, 1, 1, 2, (0, 0), (8, 0)),          # N = 136: two column tiles and a ragged one
]


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("case", CONV_GRID)
def test_conv2d_vs_float64(ops, case, precise):
    B, H, W, C, N, k, s, d, act, (xe, xo), (yo, ye) = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    xbuf = torch.randn(B, H, W, C + xe, generator=g).to(DEV)
    w = (torch.randn(N, C, k, k, generator=g) / (C * k * k) ** 0.5).double()
    scale, bias = 0.5 + torch.rand(N, generator=g), 0.1 * torch.randn(N, generator=g)
    pad = d * (k // 2)
    Ho, Wo = ops.conv2d_out(H, k, s, pad, d), ops.conv2d_out(W, k, s, pad, d)
    ybuf = torch.full((B, Ho, Wo, yo + N + ye), 7.0, device=DEV)
    with _precise(precise):
        ops.conv2d(ops.CLView(xbuf, xo, C), w.float().permute(0, 2, 3, 1).contiguous().to(DEV), ops.CLView(ybuf, yo, N),
                   k=k, stride=s, pad=pad, dil=d, scale=scale.to(DEV), bias=bias.to(DEV), act=act)
    x64 = xbuf[..., xo:xo + C].double().cpu().permute(0, 3, 1, 2)
    ref = F.conv2d(x64, w, None, s, pad, d) * scale.double()[:, None, None] + bias.double()[:, None, None]
    ref = _act64(ref, act).permute(0, 2, 3, 1)
    got = ybuf.cpu()
    e = rel(got[..., yo:yo + N], ref)
    assert e <= (5e-6 if precise else 2e-3), e
    assert (got[..., :yo] == 7).all() and (got[..., yo + N:] == 7).all()       # nothing outside the slice is written


@pytest.mark.parametrize("shape", [(2, 21, 32, 256, 4), (1, 21, 32, 256, 16), (1, 42, 64, 128, 16), (1, 3, 5, 7, 8),
                                   (2, 5, 4, 3, 1)])
def test_dwconv3x3_vs_float64(ops, shape):
    B, H, W, C, d = shape
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + d)
    x = torch.randn(B, H, W, C + 3, generator=g)
    w = torch.randn(C, 1, 3, 3, generator=g)
    y = torch.full((B, H, W, C + 2), 7.0, device=DEV)
    ops.dwconv3x3(ops.CLView(x.to(DEV), 3, C), w.reshape(C, 9).contiguous().to(DEV), ops.CLView(y, 0, C), d)
    ref = F.conv2d(x[..., 3:].double().permute(0, 3, 1, 2), w.double(), None, 1, d, d, groups=C).permute(0, 2, 3, 1)
    assert rel(y[..., :C], ref) <= 1e-6 and (y[..., C:] == 7).all()


@pytest.mark.parametrize("sizes", [((21, 32), (42, 64)), ((1, 32), (21, 32)), ((1, 1), (5, 7)), ((3, 5), (6, 10)),
                                   ((2, 2), (4, 4))])
def test_resize_bilinear_ac_vs_float64(ops, sizes):
    (Hi, Wi), (Ho, Wo) = sizes
    x = torch.randn(2, Hi, Wi, 12)
    y = torch.full((2, Ho, Wo, 20), 7.0, device=DEV)
    ops.resize_bilinear_ac(ops.CLView(x.to(DEV), 2, 10), ops.CLView(y, 4, 10))
    ref = F.interpolate(x[..., 2:].double().permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=True)
    assert rel(y[..., 4:14], ref.permute(0, 2, 3, 1)) <= 2e-6             # fp32 interpolation weights, as F.interpolate
    assert (y[..., :4] == 7).all() and (y[..., 14:] == 7).all()


def test_mean_h_vs_float64(ops):
    x = torch.randn(3, 42, 64, 40)
    y = ops.mean_h(ops.CLView(x.to(DEV), 8, 32))
    assert y.shape == (3, 1, 64, 32)
    assert rel(y, x[..., 8:].double().mean(1, keepdim=True)) <= 1e-6


@pytest.mark.parametrize("agg", [None, {"value": 0.3, "split_bin": 20}, {"value": 0.1, "split_bin": 0},
                                 {"value": 0.2, "split_bin": 100}])
def test_mask_head_vs_float64(ops, agg):
    B, mb, W, Ch, off = 2, 64, 272, 32, 8
    h = torch.randn(B, mb, W, Ch + 5) * 0.3
    w = torch.randn(2, Ch)
    mix = torch.rand(B, 2, mb + 1, W)
    for offset in (0, off):
        out = ops.vr_mask_head(ops.CLView(h.to(DEV), 5, Ch), w.to(DEV), mix.to(DEV), offset,
                               *(() if not agg else (min(agg["split_bin"], mb + 1), 1 + agg["value"] / 3,
                                                     1 + agg["value"], True)))
        m = torch.sigmoid(torch.einsum("bhwc,oc->bohw", h[..., 5:].double(), w.double()))
        m = F.pad(m, (0, 0, 0, 1), mode="replicate")
        if agg:
            sb = agg["split_bin"]
            m[:, :, :sb] = m[:, :, :sb] ** (1 + agg["value"] / 3)
            m[:, :, sb:] = m[:, :, sb:] ** (1 + agg["value"])
        ref = (m * mix.double())[..., offset:W - offset]
        assert out.shape == ref.shape and rel(out, ref) <= 1e-6


def _net(case, fp16=False):
    from easevoice_trainer_b200 import uvr5
    g = GOLD[case]
    P = O.init_params(O.param_spec(g["size"]), g["seed"])
    if fp16:
        P = {k: (v.half() if v.is_floating_point() else v) for k, v in P.items()}
    return uvr5.get_nets_model(g["n_fft"], g["size"]).to(DEV).load_state_dict(P)


def _agg(g):
    return {"value": g["agg"] / 100, "split_bin": g["split_bin"], "aggr_correction": None}


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
@pytest.mark.parametrize("case", ["small", "full"])
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


def test_reproducible_and_batch_independent(ops):
    g = GOLD["small"]
    net = _net("small")
    x = torch.cat([_predict_input(g), _predict_input(g).flip(-1)], 0)         # 4 windows
    a = net.predict(x, _agg(g))
    b = net.predict(x, _agg(g))
    assert torch.equal(a, b)
    for i in range(x.shape[0]):
        assert torch.equal(net.predict(x[i:i + 1], _agg(g)), a[i:i + 1])
    assert torch.equal(net.forward(x, _agg(g))[..., 128:-128], a)


def test_max_windows_chunking(ops):
    from easevoice_trainer_b200 import uvr5
    g = GOLD["small"]
    net = _net("small")
    spec = O.make_spec(5, 65, 700)
    data = {"window_size": 512, "tta": True}
    ref = uvr5.inference(spec, DEV, net, _agg(g), data)[0]
    for mw in (1, 3):
        assert np.array_equal(uvr5.inference(spec, DEV, net, _agg(g), data, max_windows=mw)[0], ref)


def test_from_pretrained_fp16(ops, tmp_path):
    from easevoice_trainer_b200 import uvr5
    g = GOLD["small"]
    P = O.init_params(O.param_spec(g["size"]), g["seed"])
    path = tmp_path / "vr.pth"
    torch.save({k: (v.half() if v.is_floating_point() else v) for k, v in P.items()}, path)
    net = uvr5.CascadedASPPNet.from_pretrained(str(path), n_fft=g["n_fft"])
    assert uvr5.SIZES[net.size] == uvr5.SIZES[33966]
    x = _predict_input(g)
    assert torch.equal(net.predict(x, _agg(g)), _net("small", fp16=True).predict(x, _agg(g)))
    with _precise():
        e = rel(net.predict(x, _agg(g))[..., ::g["stride"]], g["predict_out"])
    print(f"fp16 weights: rel-L2 {e:.3e}")
    assert e <= 1e-2


def test_zero_input_is_nan_like_the_reference(ops):
    from easevoice_trainer_b200 import uvr5
    net = _net("small")
    with np.errstate(invalid="ignore"):
        pred, mag, phase = uvr5.inference(np.zeros((2, 65, 40), np.complex64), DEV, net, {"value": 0.1, "split_bin": 20},
                                          {"window_size": 512, "tta": False})
    assert pred.shape == (2, 65, 40) and np.isnan(pred).all()
    assert not mag.any() and np.array_equal(phase, np.ones_like(phase))
