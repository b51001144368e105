#!/usr/bin/env python
"""Pin the BS-Roformer oracle (oracle/bs_roformer_oracle.py) against the reference's unmodified BSRoformer
(lib_v5/vr_network/bs_roformer.py) and SeparateMDXC.demix_track (uvr5/separate.py:492-574) on the CPU, and write
tests/golden/bs_roformer.pt.

rotary_embedding_torch is not installed where the pin runs: oracle/pin_uvr5.import_reference registers it as a stub, and this
script binds the oracle's functional stand-in (written from the library's documented defaults) to
bs_roformer.RotaryEmbedding before any model is built.  The reference file itself is not modified.

  1. param_spec equals BSRoformer(**cfg).state_dict(), names and shapes, and the seeded weights load strictly;
  2. the oracle's forward matches the reference's (max-abs <= 1e-5 relative to the output);
  3. the oracle's demix_track matches SeparateMDXC.demix_track, called on object.__new__(SeparateMDXC) with
     cfg = SimpleNamespace(is_half=False).
The golden keeps forward outputs at every `stride`-th sample and demix outputs at every `dstride`-th sample plus both samples
of every chunk boundary; weights and audio are regenerated from the seeds.  Cases:
  small        dim 128, depth 1, heads 2, shipped STFT and bands: forward on two 1 s stereo clips, demix on 5.5 chunks
  full         the shipped config: forward on one 2 s stereo clip, demix on 1.3 chunks
  passthrough  demix with the identity net at 0.3, 1.0, 3.3, 5.5 and 9.2 chunks: only the zeroed sample indices

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_bs_roformer.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bs_roformer_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD  # noqa: E402
from oracle.pin_uvr5 import import_reference  # noqa: E402

C = O.CHUNK
CASES = {
    "small": dict(over=dict(dim=128, depth=1, heads=2), seed=71, audio_seed=72, fwd_shape=(2, 2, 44100), stride=7,
                  demix_chunks=5.5, dstride=97),
    "full": dict(over={}, seed=81, audio_seed=82, fwd_shape=(1, 2, 88200), stride=7, demix_chunks=1.3, dstride=97),
}
PASSTHROUGH = (0.3, 1.0, 3.3, 5.5, 9.2)
PASS_SEED = 91


def config(over):
    cfg = dict(O.SHIPPED)
    cfg.update(over)
    return cfg


def demix_index(n, dstride, c=C):
    """every dstride-th sample plus the last and first sample of every chunk boundary"""
    b = np.arange(c, n, c)
    return np.unique(np.concatenate([np.arange(0, n, dstride), b - 1, b]))


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)), torch.as_tensor(np.asarray(b))
    return float((a - b).abs().max() / b.abs().max())


def pin_case(case, bs_roformer, separate):
    cfg = config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    model = bs_roformer.BSRoformer(**cfg).eval()
    sd = model.state_dict()
    assert list(sd) == list(P) and all(tuple(sd[k].shape) == tuple(v.shape) for k, v in P.items())
    model.load_state_dict(P)
    out, report = dict(case), {}
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"])
    with torch.no_grad():
        ref = model(raw)
    ora = O.forward(P, cfg, raw)
    report["forward"] = rel(ora, ref)
    assert report["forward"] <= 1e-5, report
    out["forward"] = ref[..., ::case["stride"]].contiguous()
    mix = O.make_audio(case["audio_seed"] + 100, (2, int(case["demix_chunks"] * C)))
    sep = object.__new__(separate.SeparateMDXC)
    sep.cfg = SimpleNamespace(is_half=False)
    with torch.no_grad():
        ref = sep.demix_track(model, mix, "cpu")
    ora = O.demix_track(lambda a: O.forward(P, cfg, a), mix)
    assert list(ref) == ["vocals"] and list(ora) == ["vocals"]
    report["demix"] = rel(ora["vocals"], ref["vocals"])
    assert report["demix"] <= 1e-5, report
    idx = demix_index(mix.shape[1], case["dstride"])
    out["demix_idx"] = torch.from_numpy(idx)
    out["demix"] = torch.from_numpy(np.ascontiguousarray(ref["vocals"][:, idx]))
    out["demix_zero"] = torch.from_numpy(np.nonzero((ref["vocals"] == 0).all(0))[0])
    return out, report


def pin_passthrough(separate):
    sep = object.__new__(separate.SeparateMDXC)
    sep.cfg = SimpleNamespace(is_half=False)
    out, report = {}, {}
    for k in PASSTHROUGH:
        mix = O.make_audio(PASS_SEED, (2, int(k * C)))
        with torch.no_grad():
            ref = sep.demix_track(lambda a: a, mix, "cpu")["vocals"]
        ora = O.demix_track(lambda a: a, mix)["vocals"]
        zr, zo = (np.nonzero((v == 0).all(0))[0] for v in (ref, ora))
        assert np.array_equal(zr, zo), (k, zr, zo)
        report[str(k)] = rel(ora, ref)
        assert report[str(k)] == 0.0, report
        out[str(k)] = dict(n=mix.shape[1], zero=torch.from_numpy(zr))
    return out, report


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    _, separate = import_reference()
    from src.audiokit.uvr5.lib_v5.vr_network import bs_roformer
    bs_roformer.RotaryEmbedding = O.RotaryEmbedding
    gold, report = {}, {}
    gold["passthrough"], report["passthrough"] = pin_passthrough(separate)
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, bs_roformer, separate)
    gold["keys"] = [(k, tuple(v)) for k, v in O.param_spec(config({})).items()]
    torch.save(gold, os.path.join(GOLD, "bs_roformer.pt"))
    print(report)
