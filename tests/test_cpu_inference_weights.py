"""The one strict state_dict check of the inference models (weights.check_state_dict) without a GPU: each defect it rejects,
fp16 input it accepts, and the Whisper and VR loaders rejecting a non-float tensor under a valid key."""
import os

import pytest
import torch

from oracle import pin_asr as PIN
from oracle import uvr5_echo_oracle as ECHO
from oracle import uvr5_oracle as VR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPEC = {"proj.weight": (4, 3), "proj.bias": (4,)}


def _sd(dtype=torch.float32):
    return {k: torch.zeros(s, dtype=dtype) for k, s in SPEC.items()}


def test_check_state_dict_accepts_fp16_and_fp32():
    from easevoice_trainer_b200.weights import check_state_dict
    check_state_dict(_sd(), SPEC, "net")
    check_state_dict(_sd(torch.float16), SPEC, "net")


@pytest.mark.parametrize("defect,word", [("missing", "missing"), ("unexpected", "unexpected"), ("int", "float"),
                                         ("shape", "shape")])
def test_check_state_dict_rejects(defect, word):
    from easevoice_trainer_b200.weights import check_state_dict
    sd = _sd()
    if defect == "missing":
        del sd["proj.bias"]
    elif defect == "unexpected":
        sd["proj.extra"] = torch.zeros(1)
    elif defect == "int":
        sd["proj.weight"] = torch.zeros(4, 3, dtype=torch.int64)
    else:
        sd["proj.bias"] = torch.zeros(5)
    with pytest.raises(ValueError, match=word):
        check_state_dict(sd, SPEC, "net")


def test_cached_follows_weights_and_precise_mode():
    from easevoice_trainer_b200 import lib
    from easevoice_trainer_b200.models import ParamTree
    net = ParamTree()
    net._register("proj.weight", torch.zeros(2))
    net._register("proj.stat", torch.zeros(2), buffer=True)
    builds = []

    def get():
        return net.cached("x", lambda: builds.append(1) or len(builds))
    L = lib.load()
    before = L.evk_get_precise()
    try:
        L.evk_set_precise(0)
        assert get() == 1 and get() == 1
        with torch.no_grad():
            net.P("proj.weight").add_(1)
        assert get() == 2
        net.P("proj.stat").add_(1)
        assert get() == 3
        L.evk_set_precise(1)
        assert get() == 4 and get() == 4
    finally:
        L.evk_set_precise(before)


def _int_at(sd, key):
    return dict(sd, **{key: torch.zeros(sd[key].shape, dtype=torch.int32)})


def test_whisper_rejects_int_tensor():
    from easevoice_trainer_b200 import whisper
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)
    c = gold["cases"]["m80_d2"]
    sd = PIN.make_state_dict(c["cfg"], c["seed"])
    with pytest.raises(ValueError, match="model.encoder.conv1.weight"):
        whisper.WhisperModel(c["cfg"], gold["gen"]).load_state_dict(_int_at(sd, "model.encoder.conv1.weight"))


def test_vr_nets_reject_int_tensor():
    from easevoice_trainer_b200 import uvr5
    sd = {k: torch.zeros(s) for k, s in VR.param_spec(33966).items()}
    key = next(iter(uvr5.state_dict_shapes(33966)))
    with pytest.raises(ValueError, match=key):
        uvr5.CascadedASPPNet(1024, 33966).load_state_dict(_int_at(sd, key))
    sd = ECHO.init_params(ECHO.param_spec(128, 16), 3)
    key = "stg2_high_band_net.lstm_dec2.lstm.weight_hh_l0"
    with pytest.raises(ValueError, match=key):
        uvr5.CascadedNet(128, 16).load_state_dict(_int_at(sd, key))
