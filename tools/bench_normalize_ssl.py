#!/usr/bin/env python
"""Throughput of the Normalize.ssl compute (SURVEY 8 row f3, ssl half): decoded 32 kHz samples -> int16 waveforms and HuBERT
features [1, 768, T].  Workload: the 12-layer HuBERT-base with seeded weights, 256 seeded clips of 3-12 s held as host
float32 arrays (decoding and file writes are outside the timed region; the host-to-device and device-to-host copies are in it).
GPU arms, alternated in one process: normalize_ssl.extract in ragged batches (max_batch 32) and the same library one utterance
per call (max_batch 1: B = 1 at full length).  CPU arm: the oracle restatement of the reference's per-file body
(normalize.py:151-179) on a few clips.  One JSON line with the card's name and power limit read in the same run.
   python tools/bench_normalize_ssl.py"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from easevoice_trainer_b200 import hubert, lib, ops, normalize_ssl as ns  # noqa: E402
from oracle import hubert_oracle, ssl_oracle  # noqa: E402  (seeded weights, CPU arm)

lib.init()
dev = torch.device("cuda", 0)
N, REPS = 256, 2
rng = np.random.default_rng(11)
clips = [(rng.standard_normal(int(rng.uniform(3.0, 12.0) * 32000)) * 0.1).astype(np.float32) for _ in range(N)]
m = dict(hubert_oracle.HUBERT_BASE)
P = hubert_oracle.init_params(hubert_oracle.param_spec(m), 42)
net = hubert.HubertModel()
net.load_state_dict(P)
net = net.to(dev).eval()

arms = {"batched": dict(max_batch=32), "per_utterance": dict(max_batch=1)}
for kw in arms.values():                                   # warm-up: every kernel and the allocator at these shapes
    ns.extract(net, clips[:40], **kw)
torch.cuda.synchronize()
torch.cuda.reset_peak_memory_stats()
times = {k: [] for k in arms}
outs = {}
for _ in range(REPS):
    for k, kw in arms.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs[k] = ns.extract(net, clips, **kw)
        torch.cuda.synchronize()
        times[k].append(time.perf_counter() - t0)
peak = torch.cuda.max_memory_allocated()
fa = torch.cat([o[2].flatten() for o in outs["batched"]])
fb = torch.cat([o[2].flatten() for o in outs["per_utterance"]])
wav_equal = all(np.array_equal(a[1], b[1]) for a, b in zip(outs["batched"], outs["per_utterance"]))
audio_s = sum(len(a) for a in clips) / 32000.0

# device-time split of one batch (the 32 longest clips) by CUDA events: normalisation + resampling against the HuBERT forward
grp = sorted(range(N), key=lambda i: -len(clips[i]))[:32]
n16 = [(len(clips[j]) + 1) // 2 for j in grp]
taps = torch.from_numpy(ns.resample_taps()[1]).to(dev)
x, lens_d, half_d = ns._pack(clips, grp, dev)
ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
split = []
for _ in range(3):
    ev[0].record()
    a32, a32b, status = ops.ssl_normalize(x, lens_d)
    a16 = ops.rowmask(ops.resample_poly(a32b, taps, 1, 2, 64, max(n16)).unsqueeze(-1), half_d).squeeze(-1)
    ev[1].record()
    net(a16, n16)
    ev[2].record()
    torch.cuda.synchronize()
    split.append((ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])))
wave_ms, net_ms = min(s[0] for s in split), min(s[1] for s in split)

# CPU arm: the reference's per-file computation restated (oracle), a few clips
threads = min(16, os.cpu_count() or 1)
torch.set_num_threads(threads)
n_cpu = 3
t0 = time.perf_counter()
cpu = [ssl_oracle.name2go(a, P, m) for a in clips[:n_cpu]]
cpu_s = time.perf_counter() - t0
cpu_audio = sum(len(a) for a in clips[:n_cpu]) / 32000.0
cpu_rel = max(float((o[2].double() - c["ssl"].double()).norm() / c["ssl"].double().norm()) for o, c in zip(outs["batched"], cpu))

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
best = {k: min(v) for k, v in times.items()}
print(json.dumps(dict(metric="Normalize.ssl compute (normalisation + 32->16 kHz resampling + HuBERT-base)", unit="audio-seconds/s",
                      value=audio_s / best["batched"], utterances=N, audio_seconds=audio_s,
                      batched_s=times["batched"], per_utterance_s=times["per_utterance"],
                      per_utterance_value=audio_s / best["per_utterance"], speedup=best["per_utterance"] / best["batched"],
                      rel_l2_batched_vs_per_utterance=float((fa.double() - fb.double()).norm() / fb.double().norm()),
                      int16_equal_batched_vs_per_utterance=wav_equal, peak_device_bytes=peak, card=card,
                      batch32_device_ms=dict(normalise_resample=wave_ms, hubert=net_ms,
                                             audio_seconds=sum(len(clips[j]) for j in grp) / 32000.0),
                      cpu_baseline=dict(value=cpu_audio / cpu_s, unit="audio-seconds/s", cores=threads, kind="oracle",
                                        sample=f"{n_cpu} clips, the per-file body of normalize.py:151-179",
                                        max_rel_l2_vs_batched=cpu_rel))))
