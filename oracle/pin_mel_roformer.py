#!/usr/bin/env python
"""Pin the Mel-Band Roformer oracle (oracle/mel_roformer_oracle.py) against the reference's unmodified MelBandRoformer
(lib_v5/vr_network/mel_band_roformer.py, imported with the shims mel_roformer_oracle.import_reference lists) and
SeparateMDXC.demix_track (uvr5/separate.py:492-574) on the CPU, and write tests/golden/mel_roformer.pt.

  1. for every TABLES entry, the reference's freq_indices / num_freqs_per_band / num_bands_per_freq equal the oracle's;
  2. param_spec equals MelBandRoformer(**cfg).state_dict(), names and shapes, and the seeded weights load strictly;
  3. the oracle's forward matches the reference's (max-abs <= 1e-5 relative to the output);
  4. the oracle's demix_track matches SeparateMDXC.demix_track, called on object.__new__(SeparateMDXC) with
     cfg = SimpleNamespace(is_half=False).
The golden keeps forward outputs at every `stride`-th sample and demix outputs at every `dstride`-th sample plus both samples
of every chunk boundary; weights and audio are regenerated from the seeds.  Cases:
  small    dim 128, depth 1, heads 2, 60 bands, the default STFT: forward on two 1 s stereo clips, demix on 5.5 chunks
  default  the widely distributed vocal model's config: forward on one 2 s stereo clip, demix on 1.3 chunks
  mono     dim 64, depth 2, heads 1, 24 bands at n_fft 1024, time depth 1, frequency depth 2, mask depth 1,
           match_input_audio_length: forward on two mono clips of 30 001 samples, demix on 1.2 chunks

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_mel_roformer.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mel_roformer_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD  # noqa: E402
from oracle.pin_bs_roformer import demix_index, rel  # noqa: E402

C = O.CHUNK
CASES = {
    "small": dict(over=dict(dim=128, depth=1, heads=2), seed=171, audio_seed=172, fwd_shape=(2, 2, 44100), stride=7,
                  demix_chunks=5.5, dstride=97),
    "default": dict(over={}, seed=181, audio_seed=182, fwd_shape=(1, 2, 88200), stride=7, demix_chunks=1.3, dstride=97),
    "mono": dict(over=dict(dim=64, depth=2, heads=1, stereo=False, num_bands=24, stft_n_fft=1024, stft_win_length=1024,
                           time_transformer_depth=1, freq_transformer_depth=2, mask_estimator_depth=1,
                           match_input_audio_length=True),
                 seed=191, audio_seed=192, fwd_shape=(2, 1, 30001), stride=3, demix_chunks=1.2, dstride=53),
}
# (sample_rate, n_fft, num_bands) of the band-table check
TABLES = ((44100, 2048, 60), (44100, 1024, 24), (48000, 2048, 60), (32000, 4096, 128), (22050, 512, 32), (44100, 2048, 4))


def config(over):
    cfg = dict(O.DEFAULT)
    cfg.update(over)
    return cfg


def pin_tables(M):
    out = {}
    for sr, n_fft, nb in TABLES:
        m = M.MelBandRoformer(dim=16, depth=1, heads=1, num_bands=nb, sample_rate=sr, stft_n_fft=n_fft, stft_win_length=n_fft,
                              stereo=False)
        fi, per_band, per_bin = O.band_tables(sr, n_fft, nb, False)
        assert torch.equal(m.freq_indices, fi) and torch.equal(m.num_freqs_per_band, per_band)
        assert torch.equal(m.num_bands_per_freq, per_bin)
        st = M.MelBandRoformer(dim=16, depth=1, heads=1, num_bands=nb, sample_rate=sr, stft_n_fft=n_fft, stft_win_length=n_fft,
                               stereo=True)
        assert torch.equal(st.freq_indices, O.band_tables(sr, n_fft, nb, True)[0])
        out[(sr, n_fft, nb)] = {k: v.to(torch.int32) for k, v in (("freq_indices", m.freq_indices),
                                                                  ("stereo_freq_indices", st.freq_indices),
                                                                  ("per_band", m.num_freqs_per_band),
                                                                  ("per_bin", m.num_bands_per_freq))}
    return out


def pin_case(case, M, separate):
    cfg = config(case["over"])
    P = O.init_params(O.param_spec(cfg), case["seed"])
    model = M.MelBandRoformer(**cfg).eval()
    sd = model.state_dict()
    assert list(sd) == list(P) and all(tuple(sd[k].shape) == tuple(v.shape) for k, v in P.items())
    model.load_state_dict(P)
    out, report = dict(case), {}
    raw = O.make_audio(case["audio_seed"], case["fwd_shape"])
    with torch.no_grad():
        ref = model(raw)
    ora = O.forward(P, cfg, raw)
    assert ora.shape == ref.shape, (ora.shape, ref.shape)
    report["forward"] = rel(ora, ref)
    assert report["forward"] <= 1e-5, report
    out["forward"] = ref[..., ::case["stride"]].contiguous()
    out["forward_len"] = ref.shape[-1]
    S = 2 if cfg["stereo"] else 1
    mix = O.make_audio(case["audio_seed"] + 100, (S, int(case["demix_chunks"] * C)))
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


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    M, separate = O.import_reference()
    gold, report = {}, {}
    gold["tables"] = pin_tables(M)
    for name, case in CASES.items():
        gold[name], report[name] = pin_case(case, M, separate)
        print(name, report[name], flush=True)
    gold["keys"] = [(k, tuple(v)) for k, v in O.param_spec(config({})).items()]
    torch.save(gold, os.path.join(GOLD, "mel_roformer.pt"))
    print(report)
