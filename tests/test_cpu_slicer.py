"""CPU tests of the slicing step: the oracle (oracle/slicer_oracle.py) against what the reference wrote
(tests/golden/slicer.pt, oracle/pin_slicer.py), the product's constructor and host-side silence scan against the oracle's
literal loop, the reference's quirks, and the argument errors of `write_slices`, which arrive without a device."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import slicer_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "slicer.pt"), weights_only=False)
PARAM_SETS = list(GOLD["params"].values()) + [
    dict(sr=44100, threshold=-40, min_length=5000, min_interval=30, hop_size=10, max_sil_kept=100),       # odd window: 1323
    dict(sr=8000, threshold=-20, min_length=50, min_interval=20, hop_size=20, max_sil_kept=20)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("name", list(GOLD["recordings"]))
def test_oracle_reproduces_the_reference(name):
    g = GOLD["recordings"][name]
    p = GOLD["params"][g["spec"]["params"]]
    f = so.fields(**p)
    audio = so.recording(g["spec"], p["sr"])
    assert audio.shape[0] == g["samples"]
    o = so.slice_file(audio, f, GOLD["normalize_max"], GOLD["alpha_mix"])
    assert o["failed"] == (not g["ok"]) == (name in GOLD["failed"])
    if g["rms"] is None:
        assert o["rms"] is None and not g["files"]
        return
    want = g["rms"].numpy()
    assert o["rms"].shape == want.shape and np.array_equal(np.isnan(o["rms"]), np.isnan(want))
    ok = np.isfinite(want) & (want > 0)
    assert np.all(np.abs(o["rms"][ok].astype(np.float64) - want[ok]) <= 2e-7 * want[ok])
    assert np.all(o["rms"][~ok & ~np.isnan(want)] == 0)
    assert o["tags"] == g["tags"] and o["ranges"] == g["ranges"]
    stem = name.split(".")[0]
    assert [fn for fn, _, _ in g["files"]] == ["%s_%010d_%010d.wav" % (stem, a, b) for a, b in o["ranges"]][:len(o["chunks"])]
    for (fn, n, digest), c in zip(g["files"], o["chunks"]):
        assert c.dtype == np.int16 and c.shape[0] == n and sha(c) == digest, fn
        if fn in g["full"]:
            assert np.array_equal(c, g["full"][fn].numpy())
    assert g["margins"]["threshold"] > GOLD["margin"] and g["margins"]["argmin"] > GOLD["margin"]


@pytest.mark.parametrize("p", PARAM_SETS)
def test_constructor_fields(p):
    from easevoice_trainer_b200.slicer import Slicer
    s, f = Slicer(**p), so.fields(**p)
    assert {k: getattr(s, k) for k in f} == f
    assert all(type(getattr(s, k)) is int for k in f if k != "threshold")
    for n in (0, 1, f["hop_size"] - 1, f["hop_size"], 12345, 10 * f["hop_size"]):
        assert s.num_frames(n) == so.frame_rms(np.zeros(n), f["win_size"], f["hop_size"]).shape[0]


def test_constructor_errors():
    from easevoice_trainer_b200.slicer import Slicer
    seen = set()
    for bad in (dict(sr=32000, min_length=200, min_interval=300), dict(sr=32000, hop_size=600, min_interval=700, min_length=800)):
        with pytest.raises(ValueError) as e:
            Slicer(**bad)
        assert str(e.value) == GOLD["errors"][str(sorted(bad.items()))]
        seen.add(str(e.value))
    assert len(seen) == 2


def _random_rms(rng, f, n):
    """silent and loud runs whose lengths sit on the scan's branch boundaries, with ties, exact zeros and NaN frames"""
    thr = np.float32(f["threshold"])
    marks = [1, 2, f["min_interval"], f["max_sil_kept"], 2 * f["max_sil_kept"], f["min_length"]]
    out, silent = [], bool(rng.integers(2))
    while sum(map(len, out)) < n:
        k = max(1, int(marks[rng.integers(len(marks))]) + int(rng.integers(-2, 3))) if rng.random() < 0.8 else int(rng.integers(1, 40))
        if silent:
            kind = rng.integers(4)
            v = rng.random(k) * thr * 0.99
            if kind == 1:
                v = np.round(v / thr * 3) * (thr / 4)            # few distinct values: many ties
            elif kind == 2:
                v[rng.random(k) < 0.6] = 0.0
            elif kind == 3:
                v[:] = v[0]
        else:
            v = thr * (1 + rng.random(k))
            if rng.random() < 0.1:
                v[rng.integers(k)] = thr                          # exactly the threshold is not silent
            if rng.random() < 0.05:
                v[rng.integers(k)] = np.nan
        out.append(v.astype(np.float32))
        silent = not silent
    return np.concatenate(out)[:n]


def test_run_based_scan_equals_the_literal_loop():
    from easevoice_trainer_b200.slicer import Slicer
    rng = np.random.default_rng(2024)
    small = [dict(sr=1000, threshold=-34, min_length=m, min_interval=i, hop_size=10, max_sil_kept=k)
             for m, i, k in ((400, 50, 80), (100, 100, 30), (60, 10, 10), (2000, 300, 500), (300, 40, 400))]
    count, tagged, trailing, leading = 0, 0, 0, 0
    for p in small:
        s, f = Slicer(**p), so.fields(**p)
        for trial in range(450):
            n = int(rng.integers(1, 6 * f["min_length"] + 3 * f["max_sil_kept"]))
            rms = _random_rms(rng, f, n)
            want = so.scan(rms, f)
            got = s.scan(rms)
            assert got == want, (p, trial, rms.tolist())
            assert s.ranges(got, n) == so.ranges(want, n, f["hop_size"])
            count += 1
            tagged += bool(want)
            trailing += bool(want) and want[-1][1] == n + 1
            leading += bool(want) and want[0][0] == 0
    assert count >= 2000 and tagged > count // 2 and trailing > 50 and leading > 50, (count, tagged, trailing, leading)
    # all silent, all loud, one frame
    s, f = Slicer(**small[0]), so.fields(**small[0])
    for rms in (np.zeros(300, np.float32), np.ones(300, np.float32), np.zeros(1, np.float32), np.ones(1, np.float32),
                np.full(300, np.nan, np.float32)):
        assert s.scan(rms) == so.scan(rms, f)


def test_quirks():
    f = so.fields(**so.DEFAULTS)
    rng = np.random.default_rng(5)
    # samples against frames: 400 samples are "too short", 401 are sliced
    assert so.slice_file(np.ones(400, np.float32), f)["failed"]
    o = so.slice_file((rng.standard_normal(401) * 0.2).astype(np.float32), f)
    assert not o["failed"] and o["tags"] == [] and o["ranges"] == [(0, 2 * 320)] and o["chunks"][0].shape == (401,)
    # the reported end exceeds the length; the old max divides twice
    x = (rng.standard_normal(4001) * 0.2).astype(np.float32)
    x[7] = 2.0
    m, y = so.normalize(x)
    assert m == 2.0 and y[7] == int(np.float32(np.float32(np.float32(0.5) * np.float32(0.225)) + np.float32(0.75)) * np.float32(32767))
    # digital silence: 0 / 0 -> NaN -> int16 0; NaN wins the max; values outside int16 wrap, outside int32 give 0
    assert np.array_equal(so.normalize(np.zeros(9, np.float32))[1], np.zeros(9, np.int16))
    x[9] = np.nan
    assert np.isnan(so.normalize(x)[0]) and not so.normalize(x)[1].any()
    assert np.array_equal(so.to_int16(np.array([32768.0, -32769.0, 65536.5, 3e9, -3e9, np.nan, np.inf], np.float32)),
                          np.array([-32768, 32767, 0, 0, 0, 0, 0], np.int16))
    with pytest.raises(ValueError):
        so.normalize(np.zeros(0, np.float32))
    # the empty last chunk needs a cut on the last frame, which only a NaN frame gets
    g = GOLD["recordings"]["edge_empty.wav"]
    assert g["tags"][-1][1] * so.fields(**GOLD["params"]["edge"])["hop_size"] == g["samples"] and len(g["files"]) == 1


def test_argument_errors_arrive_without_a_device(tmp_path):
    from easevoice_trainer_b200 import slicer as sl
    clips = {"a/stereo.wav": np.zeros((2, 9000), np.float32), "a/complex.wav": np.zeros(9000, np.complex64),
             "a/text.wav": np.array(["x"] * 9000), "a/long.wav": np.zeros(9001, np.float32)}
    for path in clips:
        with pytest.raises(ValueError, match=path):
            sl.write_slices([path], tmp_path, lambda f, sr: clips[f], max_samples=9000)
    s = sl.Slicer(32000)
    with pytest.raises(ValueError, match="mono"):
        s.slice(np.zeros((2, 9000), np.float32))
    with pytest.raises(ValueError, match="clip 1"):
        s.slice_batch([np.zeros(10, np.float32), np.zeros((3, 3), np.float32)])
    # files that are empty or at most min_length samples need no device either
    short = np.ones(400, np.float32)
    got = sl.write_slices(["d/none.wav", "d/short.x.wav"], tmp_path, lambda f, sr: short if "short" in f else short[:0])
    assert got == ({}, ["short"]) and not os.listdir(tmp_path)
    assert s.slice(short)[0] is short and len(s.slice(short)) == 1
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback|evk_init failed"):
            s.slice(np.ones(401, np.float32))
