#!/usr/bin/env python
"""Pin the UVR5 DeEcho / DeReverb oracle (oracle/uvr5_echo_oracle.py) against the reference's unmodified CascadedNet.predict
(lib_v5/vr_network/nets_new.py) and the SeparateVR.inference that SeparateVREcho inherits (uvr5/separate.py:198-299) on the
CPU, and write tests/golden/uvr5_deecho.pt.

  1. param_spec equals CascadedNet(n_fft, nout).state_dict(), names and shapes, and the seeded weights load strictly;
  2. the oracle's predict matches the reference's on a batch of two windows (max-abs <= 1e-5 relative to the output);
  3. the oracle's inference matches SeparateVR.inference, called on object.__new__(SeparateVREcho) (no weights file, no
     config), for every returned array.
The golden keeps the reference's outputs at every `stride`-th frame (all bins, both channels); weights and spectra are
regenerated from the seeds.  Cases:
  small     nout 16 at n_fft 128 (65 bins): 300 frames, TTA on; plus predict on two 512-frame windows
  deecho    nout 48 (the DeEcho nets) at n_fft 1344 (673 bins): 300 frames, TTA off
  dereverb  nout 64 (the DeReverb net) at n_fft 1344: 300 frames, TTA on

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_uvr5_echo.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import uvr5_echo_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD  # noqa: E402
from oracle.pin_uvr5 import import_reference  # noqa: E402  (the same stand-ins for the modules inference() never touches)

CASES = {
    "small": dict(n_fft=128, nout=16, seed=41, spec_seed=42, n_frame=300, tta=True, agg=10, predict_windows=2, stride=3),
    "deecho": dict(n_fft=1344, nout=48, seed=51, spec_seed=52, n_frame=300, tta=False, agg=10, predict_windows=0, stride=6),
    "dereverb": dict(n_fft=1344, nout=64, seed=61, spec_seed=62, n_frame=300, tta=True, agg=10, predict_windows=0, stride=6),
}


def aggressiveness(case):
    return {"value": case["agg"] / 100, "split_bin": 85, "aggr_correction": None}


def pin_case(case, nets_new, separate):
    P = O.init_params(O.param_spec(case["n_fft"], case["nout"]), case["seed"])
    model = nets_new.CascadedNet(case["n_fft"], case["nout"]).eval()
    sd = model.state_dict()
    assert list(sd) == list(P) and all(tuple(sd[k].shape) == tuple(v.shape) for k, v in P.items())
    model.load_state_dict(P)
    agg = aggressiveness(case)
    bins = case["n_fft"] // 2 + 1
    out, report = dict(case), {}
    if case["predict_windows"]:
        x = torch.from_numpy(np.abs(O.make_spec(case["spec_seed"] + 100, bins, 512 * case["predict_windows"])))
        x = x.reshape(2, bins, case["predict_windows"], 512).permute(2, 0, 1, 3).contiguous()
        x = x / x.max()
        with torch.no_grad():
            ref = model.predict(x, agg)
            ora = O.predict(P, x, agg, case["n_fft"])
        report["predict"] = float((ora - ref).abs().max() / ref.abs().max())
        assert report["predict"] <= 1e-5, report
        out["predict_out"] = ref[..., ::case["stride"]].contiguous()
    spec = O.make_spec(case["spec_seed"], bins, case["n_frame"])
    data = {"window_size": 512, "tta": case["tta"]}
    sep = object.__new__(separate.SeparateVREcho)
    with torch.no_grad():
        pred, mag, phase = sep.inference(spec, "cpu", model, agg, data)
    opred, omag, ophase = O.inference(P, spec, agg, data, case["n_fft"])
    assert np.array_equal(mag, omag) and np.array_equal(phase, ophase)
    report["inference"] = float(np.abs(opred - pred).max() / np.abs(pred).max())
    assert report["inference"] <= 1e-5, report
    out["pred"] = torch.from_numpy(np.ascontiguousarray(pred[..., ::case["stride"]]))
    out["coef"] = float(mag.max())
    return out, report


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    _, separate = import_reference()
    from src.audiokit.uvr5.lib_v5.vr_network import nets_new
    gold, report = {}, {}
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, nets_new, separate)
    torch.save(gold, os.path.join(GOLD, "uvr5_deecho.pt"))
    print(report)
