#!/usr/bin/env python
"""Pin the waveform-to-waveform VR oracle (oracle/uvr5_wave_oracle.py) against the reference's unmodified
SeparateVR.separate and SeparateVREcho.separate (uvr5/separate.py:103-196) on the CPU, and write tests/golden/uvr5_wave.pt.

The reference runs with the oracle's librosa restatement bound as the `librosa` module (librosa is not installed here), and
librosa.core.load stubbed to return the seeded clip.  separate() casts its outputs to int16 before write_output sees them,
so the float arrays are taken where they are made: spec_utils.cmb_spectrogram_to_wave is wrapped to record what it returns,
and write_output, replaced on the instance, checks that the int16 data it is given is those arrays' cast.  spec_utils' `np`
is a shim whose `ndarray` returns zero-filled arrays: cmb_spectrogram_to_wave allocates with np.ndarray and never writes
band 1's bins past crop_stop nor the top band's Nyquist bin, so the reference's output would otherwise depend on whatever
that memory held.

Cases (the parameter sets go into the golden as data):
  vr    CascadedASPPNet size 61968 (HP2 / HP3 / HP5) with 4band_v2 (SeparateVR), a 4 s stereo clip, TTA off
  echo  CascadedNet nout 48 (DeEcho) with 4band_v3 (SeparateVREcho), a 4 s mono clip, TTA on
The golden keeps x_spec_m at every 16th frame, both outputs at every 16th sample and their first and last 2048 samples.

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_uvr5_wave.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import uvr5_echo_oracle, uvr5_oracle  # noqa: E402
from oracle import uvr5_wave_oracle as W  # noqa: E402
from oracle.pin_against_reference import GOLD, REF  # noqa: E402
from oracle.pin_uvr5 import import_reference  # noqa: E402

CASES = {
    "vr": dict(net="vr", size=61968, params="4band_v2.json", seed=71, clip_seed=72, seconds=4.0, mono=False, tta=False, agg=10),
    "echo": dict(net="echo", nout=48, params="4band_v3.json", seed=81, clip_seed=82, seconds=4.0, mono=True, tta=True, agg=10),
}
SPEC_STRIDE, WAVE_STRIDE, EDGE = 16, 16, 2048


class _ZeroNdarrayNumpy(types.ModuleType):
    """numpy, except that np.ndarray(shape, dtype) returns zeros"""

    def __init__(self):
        super().__init__("numpy")

    def __getattr__(self, name):
        if name == "ndarray":
            return lambda shape, dtype=float, **kw: np.zeros(shape, dtype)
        return getattr(np, name)


def bind_librosa(clip):
    m = sys.modules["librosa"]
    m.stft = lambda y, n_fft=2048, hop_length=None, **kw: W.stft(y, n_fft, hop_length)
    m.istft = lambda stft_matrix, hop_length=None, **kw: W.istft(stft_matrix, hop_length)
    m.resample = lambda y, orig_sr, target_sr, res_type="kaiser_best", **kw: W.resample(y, orig_sr, target_sr, res_type)
    core = types.ModuleType("librosa.core")
    core.resample = m.resample
    core.load = lambda path, sr=22050, mono=True, dtype=np.float32, res_type=None, **kw: (clip.copy(), sr)
    m.core = core


def pin_case(case, separate, nets, nets_new, spec_utils, ModelParameters):
    param = ModelParameters(os.path.join(REF, "src", "audiokit", "uvr5", "lib_v5", "vr_network", "modelparams", case["params"])).param
    clip = W.make_clip(case["clip_seed"], case["seconds"], mono=case["mono"])
    bind_librosa(clip)
    n_fft = 2 * param["bins"]
    if case["net"] == "vr":
        P = uvr5_oracle.init_params(uvr5_oracle.param_spec(case["size"]), case["seed"])
        model, cls, net = nets.get_nets_model(n_fft, case["size"]), separate.SeparateVR, ("vr", False)
    else:
        P = uvr5_echo_oracle.init_params(uvr5_echo_oracle.param_spec(n_fft, case["nout"]), case["seed"])
        model, cls, net = nets_new.CascadedNet(n_fft, case["nout"]), separate.SeparateVREcho, ("echo", None)
    model.load_state_dict(P)
    model.eval()
    sep = object.__new__(cls)
    sep.input_dir, sep.output_dir = "in", "out"
    sep.mp = types.SimpleNamespace(param=param)
    sep.data = {"postprocess": False, "tta": case["tta"], "window_size": 512, "agg": case["agg"], "high_end_process": "mirroring"}
    sep.model = model
    sep.cfg = types.SimpleNamespace(device="cpu", is_half=False)
    made, got = [], {}
    cmb = spec_utils.cmb_spectrogram_to_wave
    spec_utils.cmb_spectrogram_to_wave = lambda *a, **kw: made.append(cmb(*a, **kw)) or made[-1]
    sep.write_output = lambda data, sr, name, is_vocal, extend_path=None: got.__setitem__(is_vocal, np.asarray(data))
    try:
        with torch.no_grad():
            sep.separate("clip.wav")
    finally:
        spec_utils.cmb_spectrogram_to_wave = cmb
    ref_acc, ref_voc = made
    for is_vocal, a in ((False, ref_acc), (True, ref_voc)):
        assert np.array_equal(got[is_vocal], (a * 32768).astype("int16"))
    acc, voc, x_spec_m = W.separate(P, clip, param, case["agg"], case["tta"], "mirroring", net)
    report = {k: float(np.abs(a - b).max() / np.abs(b).max()) for k, a, b in (("acc", acc, ref_acc), ("voc", voc, ref_voc))}
    assert acc.shape == ref_acc.shape and max(report.values()) <= 1e-5, report
    out = dict(case, param=param, clip_len=clip.shape[-1], l=x_spec_m.shape[2], n_out=ref_acc.shape[0],
               x_spec_m=torch.from_numpy(np.ascontiguousarray(x_spec_m[:, :, ::SPEC_STRIDE])))
    for k, a in (("acc", ref_acc), ("voc", ref_voc)):
        a = a.astype(np.float32)
        out[k] = torch.from_numpy(np.ascontiguousarray(a[::WAVE_STRIDE]))
        out[k + "_head"] = torch.from_numpy(np.ascontiguousarray(a[:EDGE]))
        out[k + "_tail"] = torch.from_numpy(np.ascontiguousarray(a[-EDGE:]))
    return out, report


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    nets, separate = import_reference()
    from src.audiokit.uvr5.lib_v5.vr_network import nets_new, spec_utils
    from src.audiokit.uvr5.lib_v5.vr_network.model_param_init import ModelParameters
    spec_utils.np = _ZeroNdarrayNumpy()
    gold, report = {"spec_stride": SPEC_STRIDE, "wave_stride": WAVE_STRIDE, "edge": EDGE}, {}
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, separate, nets, nets_new, spec_utils, ModelParameters)
    torch.save(gold, os.path.join(GOLD, "uvr5_wave.pt"))
    print(report)
