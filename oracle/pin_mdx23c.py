#!/usr/bin/env python
"""Pin the MDX23C oracle (oracle/mdx23c_oracle.py) against the reference's unmodified TFC_TDF_net
(lib_v5/vr_network/tfc_tdf_v3.py, which needs only torch) and SeparateMDXC.demix_track (uvr5/separate.py:492-574) on the
CPU, and write tests/golden/mdx23c.pt.

  1. the restated demix loop equals SeparateMDXC.demix_track at the reference's own constants (chunk 352 800, one output),
     called on object.__new__(SeparateMDXC) with cfg = SimpleNamespace(is_half=False) and a pass-through model;
  2. per case, param_spec equals TFC_TDF_net(cfg).state_dict(), names and shapes, and the seeded weights load strictly;
  3. per case, the reference's forward on a batch of chunks (which the oracle's stock-torch forward matches), and the
     restated loop over the reference's forward.
Cases:
  small    stereo, two targets, n_fft 2048, hop 512, dim_f 512, 2 subbands, 2 scales, 16 channels, growth 8, one block,
           chunk 7680: forward on two chunks and demix on 2.3 chunks, both stored whole
  mono     mono, one target (the reference's output reshaped from its [B, 2, L / 2] to [B, 1, L]), n_fft 1024, hop
           256, dim_f 256, 1 subband, 3 scales, 8 channels, growth 4, two blocks, chunk 5888: forward on two chunks and
           demix on 2.3 chunks, stored whole
  default  the 8K-FFT InstVoc configuration (mdx23c_oracle.DEFAULT): forward on one chunk, every `stride`-th sample stored

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_mdx23c.py
"""
import importlib.util
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mdx23c_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD  # noqa: E402
from oracle.pin_bs_roformer import rel  # noqa: E402

SMALL = {"audio": {"n_fft": 2048, "hop_length": 512, "dim_f": 512, "chunk_size": 7680},
         "model": {"num_subbands": 2, "num_scales": 2, "num_channels": 16, "growth": 8, "num_blocks_per_scale": 1,
                   "bottleneck_factor": 2}}
MONO = {"audio": {"n_fft": 1024, "hop_length": 256, "dim_f": 256, "chunk_size": 5888, "num_channels": 1},
        "model": {"num_subbands": 1, "num_scales": 3, "num_channels": 8, "growth": 4, "num_blocks_per_scale": 2,
                  "bottleneck_factor": 2},
        "training": {"instruments": ["vocals", "other"], "target_instrument": "vocals"}}
CASES = {
    "small": dict(over=SMALL, seed=301, audio_seed=302, batch=2, demix_chunks=2.3, stride=1),
    "mono": dict(over=MONO, seed=311, audio_seed=312, batch=2, demix_chunks=2.3, stride=1),
    "default": dict(over={}, seed=321, audio_seed=322, batch=1, demix_chunks=0, stride=16),
}


def import_reference():
    """-> the unmodified tfc_tdf_v3 module (loaded from its file: it imports only torch)"""
    ref = os.environ["EVK_REFERENCE"]
    path = os.path.join(ref, "src", "audiokit", "uvr5", "lib_v5", "vr_network", "tfc_tdf_v3.py")
    spec = importlib.util.spec_from_file_location("tfc_tdf_v3", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def pin_loop(separate):
    """the restated loop at SeparateMDXC's constants against the unmodified demix_track, pass-through model"""
    sep = object.__new__(separate.SeparateMDXC)
    sep.cfg = SimpleNamespace(is_half=False)
    net = lambda a: 0.5 * a        # noqa: E731
    out = {}
    for n in (int(2.3 * 352800), 352800 + 1000):
        mix = O.make_audio(331, (2, n))
        with torch.no_grad():
            ref = sep.demix_track(net, mix, "cpu")
        ora = O.demix_track(net, mix, 352800)
        assert list(ref) == list(ora) == ["vocals"]
        out[n] = float(np.abs(ref["vocals"] - ora["vocals"]).max())
        assert out[n] == 0.0, out
    return out


def pin_case(case, M):
    cfg = O.config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    model = M.TFC_TDF_net(O.namespace(cfg), "cpu").eval()
    sd = model.state_dict()
    assert list(sd) == list(P) and all(tuple(sd[k].shape) == tuple(v.shape) for k, v in P.items())
    model.load_state_dict(P)
    out, report = {"over": case["over"], "seed": case["seed"], "audio_seed": case["audio_seed"], "stride": case["stride"]}, {}
    S, c = cfg["audio"]["num_channels"], cfg["audio"]["chunk_size"]
    raw = O.make_audio(case["audio_seed"], (case["batch"], S, c))
    # STFT.inverse ends in reshape([*batch_dims, 2, -1]), two channels whatever num_channels is: a mono model's output
    # samples come back as [B, 2, L / 2], so they are put back as [B, 1, L] (a reshape, no value changes)
    fwd = lambda a: model(a).reshape(a.shape[0], -1, S, a.shape[-1]).squeeze(1)      # noqa: E731
    with torch.no_grad():
        ref = fwd(raw)
    report["oracle_forward"] = rel(O.forward(P, cfg, raw), ref)
    assert report["oracle_forward"] <= 1e-5, report
    out["forward"] = ref[..., ::case["stride"]].contiguous()
    out["forward_shape"] = tuple(ref.shape)
    if case["demix_chunks"]:
        mix = O.make_audio(case["audio_seed"] + 100, (S, int(case["demix_chunks"] * c)))
        with torch.no_grad():
            dem = O.demix_track(fwd, mix, c)
        out["demix_len"] = mix.shape[1]
        out["demix"] = {k: torch.from_numpy(v) for k, v in dem.items()}
        report["demix_keys"] = list(dem)
    report["forward_rms"] = float(ref.pow(2).mean().sqrt())
    return out, report


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    from oracle.pin_uvr5 import import_reference as import_uvr5
    _, separate = import_uvr5()
    M = import_reference()
    gold, report = {}, {"loop": pin_loop(separate)}
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, M)
        print(name, report[name], flush=True)
    gold["keys"] = [(k, tuple(v)) for k, v in O.param_spec(O.config({})).items()]
    torch.save(gold, os.path.join(GOLD, "mdx23c.pt"))
    print(report)
