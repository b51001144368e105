#!/usr/bin/env python
"""Pin the UVR5 VR oracle (oracle/uvr5_oracle.py) against the reference's unmodified CascadedASPPNet.predict
(lib_v5/vr_network/nets.py) and SeparateVR.inference (uvr5/separate.py:198-273) on the CPU, and write tests/golden/uvr5_vr.pt.

  1. param_spec equals get_nets_model(n_fft, size).state_dict(), names and shapes, and the seeded weights load strictly;
  2. the oracle's predict matches the reference's on a batch of two windows (max-abs <= 1e-5 relative to the output);
  3. the oracle's inference matches SeparateVR.inference, called on object.__new__(SeparateVR) (no weights file, no
     config), for every returned array.
The golden keeps the reference's outputs at every `stride`-th frame (all bins, both channels), which keeps the file small while
every window contributes; weights and spectra are regenerated from the seeds.  Cases:
  small  size 33966 (enlarge, ch 16) at n_fft 128 (65 bins): 300 frames, TTA on, agg 10, split_bin 20;
         plus predict on two 512-frame windows
  full   size 61968 (ch 32, the HP2/HP3/HP5 nets) at n_fft 1344 (673 bins): 300 frames, TTA off, split_bin 85

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_uvr5.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import uvr5_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD, REF  # noqa: E402
from oracle.ref_import import _stub  # noqa: E402

CASES = {
    "small": dict(size=33966, n_fft=128, seed=21, spec_seed=22, n_frame=300, tta=True, agg=10, split_bin=20,
                  predict_windows=2, stride=3),
    "full": dict(size=61968, n_fft=1344, seed=31, spec_seed=32, n_frame=300, tta=False, agg=10, split_bin=85,
                 predict_windows=0, stride=6),
}


def import_reference():
    """-> (nets, separate) of the unmodified reference; modules separate.py imports but inference() never touches are
    stand-ins.  src.utils.config must be one: importing the real module downloads the model weights."""
    sys.path.insert(0, REF)
    for n in ("librosa", "soundfile", "onnxruntime"):
        _stub(n)
    _stub("rotary_embedding_torch", RotaryEmbedding=object)
    _stub("pytorch_lightning", LightningModule=torch.nn.Module)
    _stub("src.utils.config", uvr5_root="", cfg=None, uvr5_params_root="", CPU="cpu", uvr5_onnx_name="",
          vocals_output="vocals", accompaniments_output="accompaniments")
    import src.audiokit.uvr5.separate as separate
    from src.audiokit.uvr5.lib_v5.vr_network import nets
    return nets, separate


def aggressiveness(case):
    return {"value": case["agg"] / 100, "split_bin": case["split_bin"], "aggr_correction": None}


def pin_case(case, nets, separate):
    P = O.init_params(O.param_spec(case["size"]), case["seed"])
    model = nets.get_nets_model(case["n_fft"], case["size"]).eval()
    sd = model.state_dict()
    assert list(sd) == list(P) and all(tuple(sd[k].shape) == tuple(v.shape) for k, v in P.items())
    model.load_state_dict(P)
    enlarge = "stg1_low_band_net.aspp.conv6.conv.0.weight" in P
    agg = aggressiveness(case)
    bins = case["n_fft"] // 2 + 1
    out, report = dict(case), {}
    if case["predict_windows"]:
        x = torch.from_numpy(np.abs(O.make_spec(case["spec_seed"] + 100, bins, 512 * case["predict_windows"])))
        x = x.reshape(2, bins, case["predict_windows"], 512).permute(2, 0, 1, 3).contiguous()
        x = x / x.max()
        with torch.no_grad():
            ref = model.predict(x, agg)
        ora = O.predict(P, x, agg, case["n_fft"], enlarge)
        report["predict"] = float((ora - ref).abs().max() / ref.abs().max())
        assert report["predict"] <= 1e-5, report
        out["predict_out"] = ref[..., ::case["stride"]].contiguous()
    spec = O.make_spec(case["spec_seed"], bins, case["n_frame"])
    data = {"window_size": 512, "tta": case["tta"]}
    sep = object.__new__(separate.SeparateVR)
    with torch.no_grad():
        pred, mag, phase = sep.inference(spec, "cpu", model, agg, data)
    opred, omag, ophase = O.inference(P, spec, agg, data, case["n_fft"], enlarge)
    assert np.array_equal(mag, omag) and np.array_equal(phase, ophase)
    report["inference"] = float(np.abs(opred - pred).max() / np.abs(pred).max())
    assert report["inference"] <= 1e-5, report
    out["pred"] = torch.from_numpy(np.ascontiguousarray(pred[..., ::case["stride"]]))
    out["coef"] = float(mag.max())
    return out, report


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    nets, separate = import_reference()
    gold, report = {}, {}
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, nets, separate)
    torch.save(gold, os.path.join(GOLD, "uvr5_vr.pt"))
    print(report)
