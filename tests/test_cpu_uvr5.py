"""UVR5 VR separator (uvr5.py) without a GPU: the oracle reproduces the golden that oracle/pin_uvr5.py took from the
reference, the state_dict key mapping, architecture inference from weight shapes and its rejections, the shape errors raised
before any GPU work, and the window arithmetic of SeparateVR.inference."""
import os

import numpy as np
import pytest
import torch

from oracle import uvr5_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_vr.pt"), weights_only=False)


def _agg(g):
    return {"value": g["agg"] / 100, "split_bin": g["split_bin"], "aggr_correction": None}


@pytest.mark.parametrize("case", ["small", "full"])
def test_oracle_matches_golden(case):
    g = _golden()[case]
    P = O.init_params(O.param_spec(g["size"]), g["seed"])
    enlarge = O.SIZES[g["size"]]["enlarge"]
    spec = O.make_spec(g["spec_seed"], g["n_fft"] // 2 + 1, g["n_frame"])
    pred, mag, phase = O.inference(P, spec, _agg(g), {"window_size": 512, "tta": g["tta"]}, g["n_fft"], enlarge)
    s = g["stride"]                                      # the golden keeps every s-th frame
    assert pred.shape == (2, g["n_fft"] // 2 + 1, g["n_frame"]) and pred[..., ::s].shape == tuple(g["pred"].shape)
    assert float(np.abs(pred[..., ::s] - g["pred"].numpy()).max()) <= 1e-6 * float(g["pred"].abs().max())
    assert float(mag.max()) == g["coef"]
    # the mask is neither saturated nor flat: the golden exercises the whole net
    m = g["pred"].numpy() / np.maximum(mag[..., ::s], 1e-30)
    assert 0.05 < float(np.median(m)) < 0.95 and float(m.std()) > 0.01
    if g["predict_windows"]:
        bins = g["n_fft"] // 2 + 1
        x = torch.from_numpy(np.abs(O.make_spec(g["spec_seed"] + 100, bins, 512 * g["predict_windows"])))
        x = x.reshape(2, bins, g["predict_windows"], 512).permute(2, 0, 1, 3).contiguous()
        out = O.predict(P, x / x.max(), _agg(g), g["n_fft"], enlarge)
        assert torch.equal(out[..., ::s], g["predict_out"])


@pytest.mark.parametrize("size", sorted(O.SIZES))
def test_key_mapping(size):
    from easevoice_trainer_b200 import uvr5
    want = {k: tuple(v) for k, v in O.param_spec(size).items() if not k.endswith("num_batches_tracked")}
    assert {k: tuple(v) for k, v in uvr5.state_dict_shapes(size).items()} == want


@pytest.mark.parametrize("size", sorted(O.SIZES))
def test_infer_size(size):
    from easevoice_trainer_b200 import uvr5
    sd = {k: torch.zeros(s) for k, s in O.param_spec(size).items()}
    got = uvr5.infer_size(sd)
    assert O.SIZES[got] == O.SIZES[size]            # 61968 / 123812 / 123821 (and 537227 / 537238) are the same net


def test_infer_size_rejects():
    from easevoice_trainer_b200 import uvr5
    sd = {k: torch.zeros(s) for k, s in O.param_spec(61968).items()}
    with pytest.raises(ValueError):
        uvr5.infer_size({k: v for k, v in sd.items() if not k.startswith("stg1_low_band_net.enc1.")})
    bad = dict(sd)
    bad["stg3_bridge.conv.0.weight"] = torch.zeros(32, 70, 1, 1)
    with pytest.raises(ValueError):
        uvr5.infer_size(bad)
    odd = {k: torch.zeros(s) for k, s in O.param_spec(61968).items()}
    odd["stg1_low_band_net.enc1.conv1.conv.0.weight"] = torch.zeros(24, 2, 3, 3)     # a width no parameter set has
    with pytest.raises(ValueError):
        uvr5.infer_size(odd)
    with pytest.raises(ValueError):                                                   # enlarge branches on the ch-32 net
        uvr5.infer_size({**sd, "stg1_low_band_net.aspp.conv6.conv.0.weight": torch.zeros(256, 1, 3, 3)})


def test_load_state_dict_folds_bn_and_rejects():
    from easevoice_trainer_b200 import uvr5
    P = O.init_params(O.param_spec(33966), 3)
    net = uvr5.get_nets_model(128, 33966).load_state_dict({k: v.half() if v.is_floating_point() else v for k, v in P.items()})
    L = net.layers["stg2_bridge"]
    p = "stg2_bridge.conv.1."
    scale = P[p + "weight"].half().double() / torch.sqrt(P[p + "running_var"].half().double() + 1e-5)
    assert torch.allclose(L["scale"].double(), scale, rtol=1e-6)
    assert torch.allclose(L["bias"].double(), P[p + "bias"].half().double() - P[p + "running_mean"].half().double() * scale,
                          rtol=1e-6, atol=1e-7)
    w = P["stg1_low_band_net.enc1.conv1.conv.0.weight"].half().float()
    assert torch.equal(net.layers["stg1_low_band_net.enc1.conv1"]["w"], w.permute(0, 2, 3, 1))
    with pytest.raises(ValueError):
        uvr5.get_nets_model(128, 33966).load_state_dict({k: v for k, v in P.items() if not k.startswith("out.")})
    with pytest.raises(ValueError):
        uvr5.get_nets_model(128, 33966).load_state_dict({**P, "extra.weight": torch.zeros(1)})
    with pytest.raises(ValueError):
        uvr5.get_nets_model(128, 12345)


def test_shape_errors_before_gpu_work():
    from easevoice_trainer_b200 import uvr5
    net = uvr5.get_nets_model(128, 33966)
    net.check_shape(512, crop=True)
    with pytest.raises(ValueError):
        net.check_shape(520, crop=True)                 # W % 16
    with pytest.raises(ValueError):
        net.check_shape(256, crop=True)                 # W <= 2 * offset
    net.check_shape(256, crop=False)
    for n_fft in (96, 130, 1346):                       # band heights 24, 32 + 33 rows, 336 + 337 rows
        with pytest.raises(ValueError):
            uvr5.get_nets_model(n_fft, 33966).check_shape(512, crop=True)
    with pytest.raises(ValueError):
        net.check_input(torch.zeros(1, 2, 64, 512), crop=True)           # 64 rows, the net wants 65
    with pytest.raises(ValueError):
        net.predict(torch.zeros(1, 2, 65, 300))
    with pytest.raises(ValueError):                                     # a spectrogram with the wrong bin count
        uvr5.inference(np.ones((2, 64, 300), np.complex64), "cpu", net, None, {"window_size": 512, "tta": False})
    with pytest.raises(ValueError):
        uvr5.inference(np.ones((2, 65, 300), np.complex64), "cpu", net, None, {"window_size": 500, "tta": False})


@pytest.mark.parametrize("width", [1, 255, 256, 257, 300, 511, 512, 16537])
def test_make_padding_and_window_counts(width):
    from easevoice_trainer_b200 import uvr5
    l, r, roi = uvr5.make_padding(width, 512, 128)
    assert (l, r, roi) == O.make_padding(width, 512, 128)
    n_window = int(np.ceil(width / roi))
    assert l + width + r >= (n_window - 1) * roi + 512           # every window lies inside the padded signal
    x = torch.arange(width, dtype=torch.float32).reshape(1, 1, width).expand(2, 3, width)
    for pl, pr, nw in ((l, r, n_window), (l + roi // 2, r + roi // 2, n_window + 1)):
        w = uvr5._windows(x, pl, pr, roi, 512, nw)
        assert w.shape == (nw, 2, 3, 512)
        xp = np.pad(x.numpy(), ((0, 0), (0, 0), (pl, pr)))
        for i in (0, nw - 1):
            assert np.array_equal(w[i].numpy(), xp[:, :, i * roi: i * roi + 512])
    assert uvr5.make_padding(100, 256, 128) == (128, 256 - 100 + 128, 256)        # roi_size == 0 -> crop_size


def test_zero_input_oracle():
    """An all-zero spectrogram: coef = 0, so x / coef is 0 / 0 and the reference's pred is NaN everywhere."""
    P = O.init_params(O.param_spec(33966), 3)
    with np.errstate(invalid="ignore"):
        pred, mag, phase = O.inference(P, np.zeros((2, 65, 40), np.complex64), {"value": 0.1, "split_bin": 20},
                                       {"window_size": 512, "tta": False}, 128, True)
    assert np.isnan(pred).all() and not mag.any() and np.array_equal(phase, np.ones_like(phase))
