#!/usr/bin/env python
"""Cost of the slicing step (AudioService.slicer without decoding and file writes): decoded 32 kHz recordings as host float32
arrays -> cut points and loudness-normalised int16 chunks on the host.  Workload: 32 seeded recordings of 3-10 minutes (bursts
of noise of 2-12 s with pauses of 0.2-1.5 s), about 3.5 hours of audio.  Needs an H100; there is no fallback.
  wall      slicer.slice_and_normalize, host arrays to host int16, synchronised: 3 repetitions after a warm-up at the same size
  kernels   CUDA-event time of evk_frame_rms and evk_slice_normalize on one resident batch over many launches, with the bytes
            each must move (frame_rms: the samples once, the RMS once; slice_normalize: the chunks' samples twice, max then
            apply, and the int16 once) over that time against the 3.35 TB/s of the H100 SXM data sheet.  Both are
            bandwidth-bound: a handful of operations per sample.
  copies    the host-to-device copy of the batch and the device-to-host copy of its int16 buffer, pageable host memory
  cpu       the oracle's restatement of the reference (float32 strided-view RMS, per-frame Python loop, numpy chunk loop) on
            this host's cores for a few of the same recordings
One JSON line, with the card's name and power limit read in the same run.
   python tools/bench_slicer.py"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from easevoice_trainer_b200 import lib, ops, slicer as sl  # noqa: E402
from easevoice_trainer_b200.normalize_ssl import _pack  # noqa: E402
from oracle import slicer_oracle as so  # noqa: E402  (CPU arm)

lib.init()
dev = torch.device("cuda", 0)
N, REPS, LAUNCHES, SR = 32, 3, 50, 32000


def recording(rng, seconds):
    parts, n = [], 0
    while n < seconds * SR:
        for dur, level in ((rng.uniform(2.0, 12.0), 0.2), (rng.uniform(0.2, 1.5), 0.001)):
            parts.append((rng.standard_normal(int(dur * SR)) * level).astype(np.float32))
            n += len(parts[-1])
    return np.concatenate(parts)[:int(seconds * SR)]


rng = np.random.default_rng(17)
clips = [recording(rng, rng.uniform(180.0, 600.0)) for _ in range(N)]
audio_s = sum(len(a) for a in clips) / SR
s = sl.Slicer(SR)


def run():
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = sl.slice_and_normalize(s, clips)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


run()                                                               # warm-up at the timed size
wall, outs = zip(*[run() for _ in range(REPS)])
n_chunks = sum(len(o["chunks"]) for o in outs[0])
same = all(np.array_equal(a, b) for o, p in zip(outs[0], outs[-1]) for a, b in zip(o["chunks"], p["chunks"]))


def events(fn, launches=LAUNCHES):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


# one resident batch: the longest recordings that fit the default budget
order = sorted(range(N), key=lambda i: -len(clips[i]))
grp = order[:max(1, sl.MAX_SAMPLES // len(clips[order[0]]))]
t0 = time.perf_counter()
x, lens_d, _ = _pack(clips, grp, dev)
torch.cuda.synchronize()
pack_h2d_s = time.perf_counter() - t0
Lm = x.shape[1]
buf = torch.from_numpy(np.zeros(x.numel() + 2 * len(grp), np.float32))
h2d_ms = events(lambda: buf.to(dev), 5)
rms_ms = events(lambda: ops.frame_rms(x, lens_d, s.win_size, s.hop_size))
rms = ops.frame_rms(x, lens_d, s.win_size, s.hop_size).cpu().numpy()
table = [(r * Lm + a, min(len(clips[j]), b) - a) for r, j in enumerate(grp)
         for a, b in s.ranges(s.scan(rms[r, :s.num_frames(len(clips[j]))]), s.num_frames(len(clips[j])))]
t = torch.tensor(table, dtype=torch.int64, device=dev)
max_len = int(t[:, 1].max())
y = torch.empty(x.numel(), dtype=torch.int16, device=dev)
c1, c2 = np.float32(0.9 * 0.25), np.float32(0.75)
norm_ms = events(lambda: ops.slice_normalize(x.view(-1), t, max_len, c1, c2, out=y))
d2h_ms = events(lambda: y.cpu(), 5)
samples = int(sum(len(clips[j]) for j in grp))
kept = int(t[:, 1].sum())
rms_bytes = 4 * samples + 4 * rms.size
norm_bytes = (4 + 4 + 2) * kept
PEAK = 3.35e12

threads = min(16, os.cpu_count() or 1)
torch.set_num_threads(threads)
n_cpu = 2
f = so.fields(**so.DEFAULTS)
t0 = time.perf_counter()
cpu = [so.slice_file(a, f, rms_fn=so.frame_rms_float32) for a in clips[:n_cpu]]
cpu_s = time.perf_counter() - t0
cpu_audio = sum(len(a) for a in clips[:n_cpu]) / SR
cpu_same = all(c["ranges"] == o["ranges"] and all(np.array_equal(a, b) for a, b in zip(c["chunks"], o["chunks"]))
               for c, o in zip(cpu, outs[0]))

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
print(json.dumps(dict(
    metric="AudioService.slicer compute (frame RMS, silence scan, chunk normalisation; host float32 -> host int16)",
    unit="audio-seconds/s", value=audio_s / min(wall), recordings=N, audio_seconds=audio_s, chunks=n_chunks, wall_s=list(wall),
    runs_identical=same, card=card,
    batch=dict(rows=len(grp), padded_samples=x.numel(), samples=samples, chunks=len(table), kept_samples=kept,
               pack_and_h2d_s=pack_h2d_s, h2d_ms=h2d_ms, h2d_GBps=4 * x.numel() / h2d_ms / 1e6,
               d2h_int16_ms=d2h_ms, d2h_GBps=2 * x.numel() / d2h_ms / 1e6,
               frame_rms_ms=rms_ms, frame_rms_GBps=rms_bytes / rms_ms / 1e6, frame_rms_share_of_hbm_peak=rms_bytes / rms_ms / 1e-3 / PEAK,
               slice_normalize_ms=norm_ms, slice_normalize_GBps=norm_bytes / norm_ms / 1e6,
               slice_normalize_share_of_hbm_peak=norm_bytes / norm_ms / 1e-3 / PEAK),
    cpu_baseline=dict(value=cpu_audio / cpu_s, unit="audio-seconds/s", cores=threads, kind="oracle", seconds=cpu_s,
                      sample=f"{n_cpu} recordings, the per-file body of audio.py:164-182", same_cuts_and_int16=cpu_same))))
