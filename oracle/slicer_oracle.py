"""CPU restatement of `AudioService.slicer` (reference src/service/audio.py:142-183) and the `Slicer` it drives
(src/audiokit/slicer/slicer.py) in numpy.

TEST INFRASTRUCTURE ONLY (tests/, oracle/pin_slicer.py, the CPU arm of tools/bench_slicer.py).  Imports nothing from the product.

  fields          slicer.py:8-31     `fields`
  frame RMS       slicer.py:149-180  `frame_rms`: float64 throughout (the reference sums float32 squares in numpy's order)
  silence scan    slicer.py:53-131   `scan`: the loop over every frame, as the reference walks it
  chunks          slicer.py:133-147  `ranges`
  normalisation   audio.py:171-178   `normalize`: float32 operations in the reference's order; int16 as x86 numpy converts
  per-file body   audio.py:164-182   `slice_file`
`recording` makes the seeded recordings of tests/golden/slicer.pt.
"""
import numpy as np

DEFAULTS = dict(sr=32000, threshold=-34, min_length=4000, min_interval=300, hop_size=10, max_sil_kept=500)


def fields(sr, threshold=-34.0, min_length=4000, min_interval=300, hop_size=10, max_sil_kept=500):
    """-> dict(threshold, hop_size, win_size, min_length, min_interval, max_sil_kept) or ValueError, as the constructor"""
    if not min_length >= min_interval >= hop_size:
        raise ValueError("The following condition must be satisfied: min_length >= min_interval >= hop_size")
    if not max_sil_kept >= hop_size:
        raise ValueError("The following condition must be satisfied: max_sil_kept >= hop_size")
    interval = sr * min_interval / 1000
    hop = round(sr * hop_size / 1000)
    return dict(threshold=10 ** (threshold / 20.0), hop_size=hop, win_size=min(round(interval), 4 * hop),
                min_length=round(sr * min_length / 1000 / hop), min_interval=round(interval / hop),
                max_sil_kept=round(sr * max_sil_kept / 1000 / hop))


def _frames(y, win, hop):
    """[frames, win] view of y padded with win // 2 zeros on both sides, one row every hop samples"""
    y = np.concatenate([np.zeros(win // 2, y.dtype), y, np.zeros(win // 2, y.dtype)])
    if y.shape[0] < win:
        return np.zeros((0, win), y.dtype)
    return np.lib.stride_tricks.sliding_window_view(y, win)[::hop]


def frame_rms(y, win, hop):
    """float64 RMS of every frame: squares and (pairwise) sums in float64"""
    x = _frames(np.asarray(y, dtype=np.float64), win, hop)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sqrt((x * x).sum(axis=1) / win)


def frame_rms_float32(y, win, hop):
    """`get_rms` the way the reference evaluates it: float32 squares of the [win, frames] strided view, numpy's mean over the
    window axis.  Used for timing and by the pin script; the tests compare against `frame_rms`."""
    x = _frames(np.asarray(y, dtype=np.float32), win, hop).T
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sqrt(np.mean(np.abs(x) ** 2, axis=0))


def scan(rms, f, windows=None):
    """sil_tags of one recording's RMS: every frame visited in turn.  windows (a list) receives the [lo, hi) of every argmin."""
    thr, msk = f["threshold"], f["max_sil_kept"]
    tags = []
    start = None                       # first frame of the silent run we are in, or that just ended
    clip = 0                           # where the current clip began
    total = rms.shape[0]

    def lowest(lo, hi):
        if windows is not None:
            windows.append((lo, min(hi, total)))
        return rms[lo:hi].argmin() + lo

    for i, v in enumerate(rms):
        if v < thr:
            if start is None:
                start = i
            continue
        if start is None:
            continue
        run = i - start
        cut = (start == 0 and i > msk) or (run >= f["min_interval"] and i - clip >= f["min_length"])
        if cut:
            if run <= msk:
                p = lowest(start, i + 1)
                tags.append((0, p) if start == 0 else (p, p))
                clip = p
            else:
                left = lowest(start, start + msk + 1)
                right = lowest(i - msk, i + 1)
                if run <= 2 * msk and start != 0:
                    mid = lowest(i - msk, start + msk + 1)
                    left, right = min(left, mid), max(right, mid)
                tags.append((0, right) if start == 0 else (left, right))
                clip = right
        start = None
    if start is not None and total - start >= f["min_interval"]:
        tags.append((lowest(start, min(total, start + msk) + 1), total + 1))
    return [(int(a), int(b)) for a, b in tags]


def ranges(tags, total, hop):
    """reported (start, end) samples of the chunks between the tags"""
    if not tags:
        return [(0, total * hop)]
    cuts = ([(0, tags[0][0])] if tags[0][0] > 0 else []) + [(a[1], b[0]) for a, b in zip(tags[:-1], tags[1:])]
    if tags[-1][1] < total:
        cuts.append((tags[-1][1], total))
    return [(a * hop, b * hop) for a, b in cuts]


def to_int16(a):
    """`a.astype(np.int16)` as numpy does it on x86-64: float -> int32 truncation (cvttss2si; NaN and out-of-range give
    INT_MIN), low 16 bits kept"""
    with np.errstate(invalid="ignore"):
        ok = np.abs(a) < 2147483648.0
        return np.where(ok, np.where(ok, a, 0).astype(np.int32), np.int32(-2 ** 31)).astype(np.int16)


def normalize(chunk, normalize_max=0.9, alpha_mix=0.25):
    """audio.py:172-178 on one chunk (not modified) -> (m, int16 samples); raises ValueError on an empty chunk, as numpy's max"""
    c = np.array(chunk, dtype=np.float32)
    m = np.abs(c).max()
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if m > 1:
            c /= m
        c = (c / m * np.float32(normalize_max * alpha_mix)) + np.float32(1 - alpha_mix) * c
        return m, to_int16(c * np.float32(32767))


def slice_file(audio, f, normalize_max=0.9, alpha_mix=0.25, rms_fn=frame_rms):
    """The body of the service's loop for one decoded file -> dict(rms, tags, ranges, chunks, failed): chunks holds the int16
    samples of the chunks that were written before a failure (a file of at most min_length samples, or an empty chunk).
    rms_fn: `frame_rms` (rounded to float32 once) or `frame_rms_float32`."""
    audio = np.asarray(audio, dtype=np.float32)
    out = dict(rms=None, tags=None, ranges=None, chunks=[], failed=False)
    if audio.shape[0] <= f["min_length"]:
        out["failed"] = True
        return out
    out["rms"] = rms_fn(audio, f["win_size"], f["hop_size"]).astype(np.float32)
    out["tags"] = scan(out["rms"], f)
    out["ranges"] = ranges(out["tags"], out["rms"].shape[0], f["hop_size"])
    for a, b in out["ranges"]:
        chunk = audio[a:min(audio.shape[0], b)]
        if chunk.shape[0] == 0:
            out["failed"] = True
            break
        out["chunks"].append(normalize(chunk, normalize_max, alpha_mix)[1])
    return out


def recording(spec, sr):
    """The seeded recordings of tests/golden/slicer.pt.  spec = dict(seed, segments=[(kind, seconds, level), ...], nan_last):
    kind "noise" is white Gaussian noise of standard deviation `level`, "peak" the same scaled so that its largest sample is
    `level`, "zero" digital silence; nan_last puts a NaN into the last sample -> float32 samples."""
    rng = np.random.default_rng(spec["seed"])
    parts = []
    for kind, seconds, level in spec["segments"]:
        n = int(round(seconds * sr))
        x = rng.standard_normal(n)
        if kind == "zero":
            x = np.zeros(n)
        elif kind == "peak":
            x = x * (level / np.abs(x).max())
        else:
            x = x * level
        parts.append(x.astype(np.float32))
    a = np.concatenate(parts)
    if spec.get("nan_last"):
        a[-1] = np.nan
    return a
