"""UVR5 DeEcho / DeReverb separator (uvr5.CascadedNet) without a GPU: the oracle reproduces the golden that
oracle/pin_uvr5_echo.py took from the reference, the state_dict key mapping, nout / nout_lstm inference from weight shapes
and the rejections, the shape errors raised before any GPU work, and `aggressiveness` being ignored."""
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import uvr5_echo_oracle as O
from oracle import uvr5_oracle as VR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_deecho.pt"), weights_only=False)


def _agg(g):
    return {"value": g["agg"] / 100, "split_bin": 85, "aggr_correction": None}


@pytest.mark.parametrize("case", ["small", "deecho", "dereverb"])
def test_oracle_matches_golden(case):
    g = _golden()[case]
    P = O.init_params(O.param_spec(g["n_fft"], g["nout"]), g["seed"])
    bins = g["n_fft"] // 2 + 1
    spec = O.make_spec(g["spec_seed"], bins, g["n_frame"])
    pred, mag, phase = O.inference(P, spec, _agg(g), {"window_size": 512, "tta": g["tta"]}, g["n_fft"])
    s = g["stride"]                                      # the golden keeps every s-th frame
    assert pred.shape == (2, bins, g["n_frame"]) and pred[..., ::s].shape == tuple(g["pred"].shape)
    assert float(np.abs(pred[..., ::s] - g["pred"].numpy()).max()) <= 1e-6 * float(g["pred"].abs().max())
    assert float(mag.max()) == g["coef"]
    # the mask is neither saturated nor flat: the golden exercises the whole net
    m = g["pred"].numpy() / np.maximum(mag[..., ::s], 1e-30)
    assert 0.05 < float(np.median(m)) < 0.95 and float(m.std()) > 0.01
    if g["predict_windows"]:
        x = torch.from_numpy(np.abs(O.make_spec(g["spec_seed"] + 100, bins, 512 * g["predict_windows"])))
        x = x.reshape(2, bins, g["predict_windows"], 512).permute(2, 0, 1, 3).contiguous()
        with torch.no_grad():
            out = O.predict(P, x / x.max(), _agg(g), g["n_fft"])
        assert torch.equal(out[..., ::s], g["predict_out"])


@pytest.mark.parametrize("n_fft,nout,nout_lstm", [(128, 16, 128), (1344, 48, 128), (1344, 64, 128), (256, 32, 128)])
def test_key_mapping_and_config_inference(n_fft, nout, nout_lstm):
    from easevoice_trainer_b200 import uvr5
    spec = O.param_spec(n_fft, nout, nout_lstm)
    want = {k: tuple(v) for k, v in spec.items() if not k.endswith("num_batches_tracked")}
    assert {k: tuple(v) for k, v in uvr5.echo_state_dict_shapes(n_fft, nout, nout_lstm).items()} == want
    sd = {k: torch.zeros(s) for k, s in spec.items()}
    assert uvr5.infer_echo_config(sd) == (nout, nout_lstm)
    net = uvr5.CascadedNet(n_fft, nout, nout_lstm)
    assert (net.max_bin, net.output_bin, net.nin_lstm, net.offset) == (n_fft // 2, n_fft // 2 + 1, n_fft // 4, 64)


def test_load_state_dict_folds_and_lays_out():
    from easevoice_trainer_b200 import uvr5
    P = O.init_params(O.param_spec(128, 16), 3)
    net = uvr5.CascadedNet(128, 16).load_state_dict({k: v.half() if v.is_floating_point() else v for k, v in P.items()})
    h = {k: v.half().double() for k, v in P.items() if v.is_floating_point()}
    # BatchNorm2d folding
    p = "stg2_low_band_net.1.conv.1."
    scale = h[p + "weight"] / torch.sqrt(h[p + "running_var"] + 1e-5)
    L = net.layers["stg2_low_band_net.1"]
    assert torch.allclose(L["scale"].double(), scale, rtol=1e-6)
    assert torch.allclose(L["bias"].double(), h[p + "bias"] - h[p + "running_mean"] * scale, rtol=1e-6, atol=1e-7)
    # stage-3 enc1 reads [x | 0 0 | aux1 (4) | aux2 (8)]: 16 columns, zeros at 2 and 3
    w = net.layers["stg3_full_band_net.enc1"]["w"]
    ref = P["stg3_full_band_net.enc1.conv.0.weight"].half().float().permute(0, 2, 3, 1)
    assert w.shape == (16, 3, 3, 16) and not w[..., 2:4].any()
    assert torch.equal(w[..., [0, 1] + list(range(4, 16))], ref)
    # dec1 of stg1_high (ch 4) reads [e1 (4) | up(dec2) (8) | up(lstm) (1) | 0 0 0]
    w = net.layers["stg1_high_band_net.dec1.conv1"]["w"]
    ref = P["stg1_high_band_net.dec1.conv1.conv.0.weight"].half().float().permute(0, 2, 3, 1)   # [up (8), lstm (1), e1 (4)]
    assert w.shape == (4, 3, 3, 16) and not w[..., 13:].any()
    assert torch.equal(w[..., :4], ref[..., 9:]) and torch.equal(w[..., 4:13], ref[..., :9])
    # LSTM: both biases summed, BatchNorm1d folded into the dense layer
    q = "stg3_full_band_net.lstm_dec2"
    L = net.layers[q]
    b = torch.cat([h[f"{q}.lstm.bias_ih_l0{s}"] + h[f"{q}.lstm.bias_hh_l0{s}"] for s in ("", "_reverse")])
    assert L["w_ih"].shape == (8 * 64, 32) and L["w_hh"].shape == (2, 256, 64)
    assert torch.allclose(L["b"].double(), b, rtol=1e-6, atol=1e-7)
    sc = h[q + ".dense.1.weight"] / torch.sqrt(h[q + ".dense.1.running_var"] + 1e-5)
    assert torch.allclose(L["w_d"].double(), h[q + ".dense.0.weight"] * sc[:, None], rtol=1e-6, atol=1e-7)


def test_rejects_foreign_truncated_and_misshaped():
    from easevoice_trainer_b200 import uvr5
    P = O.init_params(O.param_spec(128, 16), 3)
    vr = {k: torch.zeros(s) for k, s in VR.param_spec(33966).items()}
    with pytest.raises(ValueError):                                      # a CascadedASPPNet state_dict
        uvr5.infer_echo_config(vr)
    with pytest.raises(ValueError):
        uvr5.CascadedNet(128, 16).load_state_dict(vr)
    with pytest.raises(ValueError):                                      # truncated
        uvr5.CascadedNet(128, 16).load_state_dict({k: v for k, v in P.items() if not k.startswith("stg3_full_band_net.dec1")})
    with pytest.raises(ValueError):                                      # unexpected key
        uvr5.CascadedNet(128, 16).load_state_dict({**P, "extra.weight": torch.zeros(1)})
    bad = dict(P)
    bad["stg2_high_band_net.lstm_dec2.lstm.weight_hh_l0"] = torch.zeros(128, 31)
    with pytest.raises(ValueError):                                      # mis-shaped
        uvr5.CascadedNet(128, 16).load_state_dict(bad)
    with pytest.raises(ValueError):                                      # right net, wrong n_fft (LSTM input size)
        uvr5.CascadedNet(256, 16).load_state_dict(P)
    with pytest.raises(ValueError):                                      # hidden sizes the recurrence kernel lacks
        uvr5.CascadedNet(128, 16, nout_lstm=256)
    with pytest.raises(ValueError):
        uvr5.CascadedNet(128, 16, nout_lstm=64)
    uvr5.CascadedNet(128, 16).load_state_dict(P)                         # and the full set loads


def test_shape_errors_before_gpu_work():
    from easevoice_trainer_b200 import uvr5
    net = uvr5.CascadedNet(128, 16)
    net.check_shape(512, crop=True)
    net.check_shape(144, crop=True)
    with pytest.raises(ValueError):
        net.check_shape(520, crop=True)                 # W % 16
    with pytest.raises(ValueError):
        net.check_shape(128, crop=True)                 # W <= 2 * offset
    net.check_shape(128, crop=False)
    for n_fft in (96, 130, 1346):                       # band heights 24, 32 + 33 rows, 336 + 337 rows
        with pytest.raises(ValueError):
            uvr5.CascadedNet(n_fft, 16).check_shape(512, crop=True)
    with pytest.raises(ValueError):
        net.check_input(torch.zeros(1, 2, 64, 512), crop=True)           # 64 rows, the net wants 65
    with pytest.raises(ValueError):
        net.predict(torch.zeros(1, 2, 65, 300))
    with pytest.raises(ValueError):                                     # no weights loaded
        net.predict(torch.zeros(1, 2, 65, 512))
    with pytest.raises(ValueError):                                     # a spectrogram with the wrong bin count
        uvr5.inference(np.ones((2, 64, 300), np.complex64), "cpu", net, None, {"window_size": 512, "tta": False})
    with pytest.raises(ValueError):
        uvr5.inference(np.ones((2, 65, 300), np.complex64), "cpu", net, None, {"window_size": 500, "tta": False})


def test_window_arithmetic_offset_64():
    from easevoice_trainer_b200 import uvr5
    net = uvr5.CascadedNet(1344, 48)
    l, r, roi = uvr5.make_padding(16538, 512, net.offset)
    assert (l, roi) == (64, 384) and int(np.ceil(16538 / roi)) == 44


def test_predict_ignores_aggressiveness():
    from easevoice_trainer_b200 import uvr5
    assert "aggressiveness" in inspect.signature(uvr5.CascadedNet.predict).parameters
    P = O.init_params(O.param_spec(128, 16), 3)
    x = torch.rand(1, 2, 65, 256)
    with torch.no_grad():
        a = O.predict(P, x, None, 128)
        b = O.predict(P, x, {"value": 0.9, "split_bin": 10, "aggr_correction": None}, 128)
    assert torch.equal(a, b)
