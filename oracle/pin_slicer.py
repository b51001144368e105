#!/usr/bin/env python
"""Run the reference's unmodified `Slicer` (src/audiokit/slicer/slicer.py) and the loop `AudioService.slicer` runs around it
(src/service/audio.py:164-182) on seeded recordings on the CPU, check oracle/slicer_oracle.py against them, and write
tests/golden/slicer.pt.

What is substituted, and nothing else: `load_audio` returns the seeded recording (decoding is not part of the contract).

Recordings (slicer_oracle.recording; bursts of white noise at 0.2 with pauses of noise at 0.001 or digital silence):
  branches     leading pause of 0.8 s (leading silence, <= 2 max_sil_kept), pauses of 0.4 s (<= max_sil_kept), 0.8 s
               (<= 2 max_sil_kept) and 1.5 s (longer), trailing pause of 1 s
  lead_long    leading pause of 1.5 s (> 2 max_sil_kept), a pause of digital silence (argmin ties at exactly 0)
  no_tag       a short leading pause and no cut: one chunk
  silent       5000 samples of digital silence: one chunk with max 0, every sample int16(NaN) = 0
  loud         chunks with max 1.7 and 1.3, divided twice
  short        300 samples: `slice` returns `[waveform]`, the service's loop fails on it
  alt_*        sr = 16000, hop_size = 20, min_interval = 50: a window of 800 samples = 2.5 hops
  edge_empty   min_interval = hop_size (window = hop), a length that is a multiple of hop and a NaN in the last sample: only the
               last frame is NaN, the cut lands on it, the first chunk is written (all 0) and the empty last chunk fails
The device RMS is the float64 value rounded once rather than numpy's float32 mean, so every decision of a golden recording
must not hang on the last digits: each `rms < threshold` is off the threshold by more than MARGIN relative, and in each argmin
window the runner-up exceeds the minimum by more than MARGIN relative unless both are exactly 0 (first index wins on both
sides).  A recording that fails this is drawn again with another seed; the margins found are recorded.

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_slicer.py
"""
import hashlib
import importlib.util
import os
import sys
import tempfile

import numpy as np
import torch
from scipy.io import wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import slicer_oracle as so  # noqa: E402

REF = os.environ.get("EVK_REFERENCE", "")
GOLD = os.path.join(ROOT, "tests", "golden")
MARGIN = 1e-5
NORMALIZE_MAX, ALPHA_MIX = 0.9, 0.25
PARAMS = dict(default=dict(so.DEFAULTS),
              alt=dict(sr=16000, threshold=-34, min_length=2000, min_interval=50, hop_size=20, max_sil_kept=300),
              edge=dict(sr=32000, threshold=-34, min_length=1000, min_interval=10, hop_size=10, max_sil_kept=500))
N, Q, Z, P = "noise", "noise", "zero", "peak"
LOUD, QUIET = 0.2, 0.001
RECORDINGS = [
    dict(name="branches.wav", params="default", seed=101, segments=[
        (Q, 0.8, QUIET), (N, 5.003, LOUD), (Q, 0.4, QUIET), (N, 5.0, LOUD), (Q, 0.8, QUIET), (N, 5.0, LOUD), (Q, 1.5, QUIET),
        (N, 5.0, LOUD), (Q, 1.0, QUIET)]),
    dict(name="lead_long.flac", params="default", seed=102, segments=[
        (Q, 1.5, QUIET), (N, 4.5, LOUD), (Z, 0.6, 0), (N, 4.5017, LOUD)]),
    dict(name="no_tag.wav", params="default", seed=103, segments=[(Q, 0.4, QUIET), (N, 2.6, LOUD)]),
    dict(name="silent.wav", params="default", seed=104, segments=[(Z, 0.15625, 0)]),
    dict(name="loud.take2.wav", params="default", seed=105, segments=[(P, 5.0, 1.7), (Q, 0.6, QUIET), (P, 5.0, 1.3)]),
    dict(name="short.wav", params="default", seed=106, segments=[(N, 0.009375, LOUD)]),
    dict(name="alt_branches.wav", params="alt", seed=107, segments=[
        (Q, 0.5, QUIET), (N, 3.0, LOUD), (Q, 0.2, QUIET), (N, 3.0, LOUD), (Q, 0.5, QUIET), (N, 3.0, LOUD), (Q, 1.0, QUIET),
        (N, 2.0101, LOUD)]),
    dict(name="alt_trailing.wav", params="alt", seed=108, segments=[(N, 2.5, LOUD), (Q, 0.7, QUIET)]),
    dict(name="edge_empty.wav", params="edge", seed=109, nan_last=True, segments=[(N, 2.0, LOUD), (Q, 0.2, QUIET)]),
]
FULL = ("no_tag.wav", "edge_empty.wav")          # recordings whose int16 chunks are stored whole


def import_slicer():
    spec = importlib.util.spec_from_file_location("ref_slicer", os.path.join(REF, "src/audiokit/slicer/slicer.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.Slicer


def service_loop(slicer, name, audio, out_dir, sr):
    """audio.py:165-182 for one file -> True if the file reached `data`"""
    name = name.split(".")[0]
    try:
        if audio.shape[0] == 0:
            return False
        for chunk, start, end in slicer.slice(audio):
            nor_max = np.abs(chunk).max()
            if nor_max > 1:
                chunk /= nor_max
            chunk = (chunk / nor_max * (NORMALIZE_MAX * ALPHA_MIX)) + (1 - ALPHA_MIX) * chunk
            wavfile.write(os.path.join(out_dir, "%s_%010d_%010d.wav" % (name, start, end)), sr, (chunk * 32767).astype(np.int16))
        return True
    except Exception as e:
        print(f"  {name}: slice failed: {type(e).__name__}: {e}")
        return False


def margins(rms, f):
    """-> (least relative distance of a frame's RMS from the threshold, least relative gap between the two lowest frames of an
    argmin window, windows skipped because they hold a NaN or tie at exactly 0)"""
    ok = np.isfinite(rms)
    thr = np.float64(f["threshold"])
    m_thr = float(np.min(np.abs(rms[ok].astype(np.float64) - thr) / thr)) if ok.any() else float("inf")
    windows, m_arg, skipped = [], float("inf"), 0
    so.scan(rms, f, windows)
    for lo, hi in windows:
        w = np.sort(rms[lo:hi].astype(np.float64))
        if hi - lo < 2:
            continue
        if np.isnan(w).any() or w[1] == 0:
            skipped += 1
            continue
        m_arg = min(m_arg, float((w[1] - w[0]) / w[1]))
    return m_thr, m_arg, skipped


def pin_one(Slicer, rec, tmp):
    p = PARAMS[rec["params"]]
    f = so.fields(**p)
    ref = Slicer(**p)
    assert {k: getattr(ref, k) for k in f} == f, (f, vars(ref))
    audio = so.recording(rec, p["sr"])
    out_dir = os.path.join(tmp, rec["name"] + ".d")
    os.makedirs(out_dir)
    ok = service_loop(ref, rec["name"], audio.copy(), out_dir, p["sr"])
    g = dict(spec=rec, samples=int(audio.shape[0]), ok=ok, rms=None, tags=None, ranges=None, files=[], margins=None, full={})
    files = sorted(os.listdir(out_dir))
    for fn in files:
        sr, w = wavfile.read(os.path.join(out_dir, fn))
        assert sr == p["sr"] and w.dtype == np.int16
        g["files"].append((fn, int(w.shape[0]), hashlib.sha256(w.tobytes()).hexdigest()))
        if rec["name"] in FULL:
            g["full"][fn] = torch.from_numpy(w.copy())
    o = so.slice_file(audio, f, NORMALIZE_MAX, ALPHA_MIX)
    assert o["failed"] == (not ok), rec["name"]
    if o["rms"] is None:
        assert not files
        return g, True
    rms = ref.get_rms(y=audio, frame_length=ref.win_size, hop_length=ref.hop_size).squeeze(0)
    assert rms.dtype == np.float32 and rms.shape == o["rms"].shape
    assert np.array_equal(rms, so.frame_rms_float32(audio, f["win_size"], f["hop_size"]), equal_nan=True)
    assert np.array_equal(np.isnan(rms), np.isnan(o["rms"]))
    fin = np.isfinite(rms) & (rms > 0)
    rel = float(np.max(np.abs(o["rms"][fin].astype(np.float64) - rms[fin]) / rms[fin])) if fin.any() else 0.0
    m_thr, m_arg, skipped = margins(rms, f)
    g["margins"] = dict(threshold=m_thr, argmin=m_arg, windows_skipped=skipped, rms_rel_oracle_vs_reference=rel)
    if not (m_thr > MARGIN and m_arg > MARGIN):
        return g, False
    tags = so.scan(rms, f)
    assert tags == o["tags"], rec["name"]                               # float64 RMS and numpy's decide alike
    want = ["%s_%010d_%010d.wav" % (rec["name"].split(".")[0], a, b) for a, b in o["ranges"]][:len(o["chunks"])]
    assert want == files, (want, files)
    for (fn, n, sha), c in zip(g["files"], o["chunks"]):
        assert n == c.shape[0] and sha == hashlib.sha256(c.tobytes()).hexdigest(), fn
    g.update(rms=torch.from_numpy(rms.copy()), tags=tags, ranges=o["ranges"])
    return g, True


def main():
    Slicer = import_slicer()
    gold = dict(numpy=np.__version__, params=PARAMS, normalize_max=NORMALIZE_MAX, alpha_mix=ALPHA_MIX, margin=MARGIN,
                recordings={}, written=[], failed=[])
    for bad in (dict(sr=32000, min_length=200, min_interval=300), dict(sr=32000, hop_size=600, min_interval=700, min_length=800)):
        for make in (Slicer, so.fields):
            try:
                make(**bad)
                raise AssertionError(bad)
            except ValueError as e:
                gold.setdefault("errors", {})[str(sorted(bad.items()))] = str(e)
    with tempfile.TemporaryDirectory() as tmp:
        for rec in RECORDINGS:
            rec = dict(rec)
            for attempt in range(20):
                g, ok = pin_one(Slicer, rec, os.path.join(tmp, str(attempt)))
                if ok:
                    break
                print(f"  {rec['name']}: margins {g['margins']} too small with seed {rec['seed']}, drawing again")
                rec["seed"] += 1000
            assert ok, rec["name"]
            gold["recordings"][rec["name"]] = g
            (gold["written"] if g["ok"] else gold["failed"]).append(rec["name"])
            print(rec["name"], "ok" if g["ok"] else "FAILED", "tags", g["tags"], "files", len(g["files"]), "margins", g["margins"])
    R = gold["recordings"]
    assert gold["failed"] == ["short.wav", "edge_empty.wav"], gold["failed"]
    assert len(R["edge_empty.wav"]["files"]) == 1 and not R["short.wav"]["files"]
    assert R["no_tag.wav"]["tags"] == [] and R["silent.wav"]["tags"] == [] and len(R["silent.wav"]["files"]) == 1
    t = R["branches.wav"]["tags"]
    f = so.fields(**PARAMS["default"])
    assert len(t) == 5 and t[0][0] == 0 and t[1][0] == t[1][1] and t[-1][1] == R["branches.wav"]["rms"].shape[0] + 1, t
    assert R["lead_long.flac"]["tags"][0][0] == 0 and R["lead_long.flac"]["tags"][0][1] >= 2 * f["max_sil_kept"]
    assert R["lead_long.flac"]["margins"]["windows_skipped"] > 0
    torch.save(gold, os.path.join(GOLD, "slicer.pt"))
    print("wrote", os.path.join(GOLD, "slicer.pt"), os.path.getsize(os.path.join(GOLD, "slicer.pt")), "bytes")


if __name__ == "__main__":
    main()
