"""GPU tests of the slicing step (`pytest -m gpu`): evk_frame_rms against float64, evk_slice_normalize bit for bit against
numpy, and `slice_batch` / `write_slices` against what the reference wrote (tests/golden/slicer.pt, oracle/pin_slicer.py)."""
import hashlib
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import slicer_oracle as so

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "slicer.pt"), weights_only=False)
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init()
    return ops


def _rms(ops, rows, win, hop):
    L = max(len(r) for r in rows)
    x = np.zeros((len(rows), L), np.float32)
    for r, a in enumerate(rows):
        x[r, :len(a)] = a
    lens = torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV)
    return ops.frame_rms(torch.from_numpy(x).to(DEV), lens, win, hop).cpu().numpy()


def _within_one_ulp(got, want64):
    """got float32 against the float64 value: NaN or Inf where it is, else |got - want| <= the spacing of float32 at want"""
    nan = ~np.isfinite(want64)
    assert np.array_equal(np.isnan(got), np.isnan(want64)) and np.array_equal(np.isinf(got), np.isinf(want64))
    w32 = want64[~nan].astype(np.float32)
    ulp = np.maximum(np.spacing(np.abs(w32)), np.spacing(np.abs(got[~nan]))).astype(np.float64)
    err = np.abs(got[~nan].astype(np.float64) - want64[~nan])
    assert np.all(err <= ulp), float(np.max(err / ulp))


@pytest.mark.parametrize("win,hop", [(1280, 320), (800, 320), (1323, 441), (320, 320), (100, 160), (64, 1)])
def test_frame_rms_within_one_ulp_of_float64(ops, win, hop):
    rng = np.random.default_rng(win + hop)
    lens = [50000, 49999, 3 * hop, 3 * hop + 1, hop - 1 if hop > 1 else 1, max(1, win // 2 - 1), 1, 20 * 64 * hop + 7]
    rows = [(rng.standard_normal(n) * rng.choice([1e-3, 0.2, 3.0])).astype(np.float32) for n in lens]
    rows[0][:20000] *= np.float32(1e-4)                       # a quiet passage before a loud one
    rows[1][31000] = np.nan
    rows[2][1] = np.inf
    got = _rms(ops, rows, win, hop)
    assert got.shape[1] == 1 + (max(lens) + 2 * (win // 2) - win) // hop
    for r, a in enumerate(rows):
        want = so.frame_rms(a, win, hop)
        assert (got[r, want.shape[0]:] == 0).all(), r                                     # frames past the row's end
        _within_one_ulp(got[r, :want.shape[0]], want)
        assert np.isnan(got[r]).any() == (r == 1) and np.isinf(got[r]).any() == (r == 2)
        alone = _rms(ops, [a], win, hop)[0]                                               # the same bits alone
        assert np.array_equal(alone.view(np.int32), got[r, :alone.shape[0]].view(np.int32)), r


def test_frame_rms_on_the_golden(ops):
    for name, g in GOLD["recordings"].items():
        if g["rms"] is None:
            continue
        p = GOLD["params"][g["spec"]["params"]]
        f = so.fields(**p)
        a = so.recording(g["spec"], p["sr"])
        got = _rms(ops, [a], f["win_size"], f["hop_size"])[0]
        assert got.shape == g["rms"].shape
        _within_one_ulp(got, so.frame_rms(a, f["win_size"], f["hop_size"]))
        ref = g["rms"].numpy()
        ok = np.isfinite(ref) & (ref > 0)
        assert np.all(np.abs(got[ok].astype(np.float64) - ref[ok]) <= 2e-7 * ref[ok]), name


def test_frame_rms_rejects_bad_arguments(ops):
    x = torch.zeros(1, 1000, device=DEV)
    lens = torch.tensor([1000], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="frame_rms"):
        ops.frame_rms(x, lens, 65 * 4, 4)
    with pytest.raises(RuntimeError, match="frame_rms"):
        ops.frame_rms(x, lens, 0, 4)


def _normalize(ops, chunks, pad=3, c1=0.9 * 0.25, c2=0.75):
    """chunks laid out one after the other with `pad` untouched samples in between -> (int16 per chunk, m, status)"""
    table, parts, off = [], [], 0
    for c in chunks:
        parts += [np.full(pad, 7.0, np.float32), c]
        table.append((off + pad, len(c)))
        off += pad + len(c)
    x = torch.from_numpy(np.concatenate(parts)).to(DEV)
    t = torch.tensor(table, dtype=torch.int64, device=DEV)
    out = torch.full(x.shape, 12345, dtype=torch.int16, device=DEV)
    y, m, status = ops.slice_normalize(x, t, max(len(c) for c in chunks), np.float32(c1), np.float32(c2), out=out)
    y = y.cpu().numpy()
    keep = np.ones(y.shape[0], bool)
    for o, n in table:
        keep[o:o + n] = False
    assert (y[keep] == 12345).all()                                     # nothing outside the chunks is written
    return [y[o:o + n] for o, n in table], m.cpu().numpy(), status.cpu().tolist()


def test_slice_normalize_bit_identical_to_numpy(ops):
    from easevoice_trainer_b200 import slicer as sl
    rng = np.random.default_rng(9)
    chunks = [(rng.standard_normal(n) * s).astype(np.float32) for n, s in
              ((128000, 0.2), (4001, 0.05), (1, 0.3), (70001, 0.9), (33333, 2.5), (3_000_001, 0.2))]
    chunks.append(np.zeros(5000, np.float32))                                              # m == 0
    chunks.append(chunks[1].copy()); chunks[-1][17] = np.nan                               # NaN wins the max
    chunks.append(chunks[1].copy()); chunks[-1][3] = np.inf
    chunks.append(chunks[1].copy()); chunks[-1][-1] = -1.5                                 # m > 1 from a negative last sample
    assert np.abs(chunks[3]).max() > 1 and np.abs(chunks[4]).max() > 1
    got, m, status = _normalize(ops, chunks)
    want_status = [sl.SLICE_OK] * 6 + [sl.SLICE_SILENT, sl.SLICE_NONFINITE, sl.SLICE_NONFINITE, sl.SLICE_OK]
    assert status == want_status
    for i, c in enumerate(chunks):
        wm, wy = so.normalize(c)
        assert np.array_equal(np.float32(wm).view(np.int32), m[i].view(np.int32)) or (np.isnan(wm) and np.isnan(m[i])), i
        assert np.array_equal(got[i], wy), i
    assert not got[6].any() and not got[7].any()
    # a mix that wraps int16 and one that leaves int32
    for c1, c2 in ((3.0, 0.75), (1e6, 0.75)):
        got, _, _ = _normalize(ops, chunks[:2], c1=c1, c2=c2)
        for g, c in zip(got, chunks[:2]):
            with np.errstate(invalid="ignore"):
                want = so.to_int16(((c / np.abs(c).max() * np.float32(c1)) + np.float32(c2) * c) * np.float32(32767))
            assert np.array_equal(g, want)
            assert (np.abs(((c / np.abs(c).max() * np.float32(c1)) + np.float32(c2) * c) * np.float32(32767)) > 32767).any()


def _load_audio(sr_want):
    def load(path, sr):
        assert sr == sr_want
        if os.path.basename(path) == "nothing.wav":
            return np.zeros(0, np.float32)
        r, a = wavfile.read(path)
        assert r == sr and a.dtype == np.float32
        return a
    return load


@pytest.mark.parametrize("pset", list(GOLD["params"]))
def test_slice_batch_and_write_slices_against_the_golden(ops, tmp_path, pset):
    from easevoice_trainer_b200 import slicer as sl
    p = GOLD["params"][pset]
    recs = {n: g for n, g in GOLD["recordings"].items() if g["spec"]["params"] == pset}
    src = tmp_path / "src"
    os.makedirs(src)
    files, clips = [], []
    for n, g in recs.items():
        a = so.recording(g["spec"], p["sr"])
        wavfile.write(src / n, p["sr"], a)                                                 # float32 WAV
        files.append(str(src / n))
        clips.append(a)
    files.append(str(src / "nothing.wav"))                                                 # empty audio: skipped
    s = sl.Slicer(**p)
    for max_samples in (sl.MAX_SAMPLES, max(len(a) for a in clips)):                       # one batch, one row per batch
        for (n, g), a, res in zip(recs.items(), clips, s.slice_batch(clips, max_samples=max_samples)):
            if g["rms"] is None:
                assert res is None
                assert s.slice(a)[0] is a
                continue
            assert res[1] == g["tags"] and res[0] == g["ranges"], n
            chunks = s.slice(a)
            assert [(c[1], c[2]) for c in chunks] == g["ranges"]
            assert all(np.shares_memory(c[0], a) or c[0].size == 0 for c in chunks)
    kw = dict(threshold=p["threshold"], min_length=p["min_length"], min_interval=p["min_interval"], hop_size=p["hop_size"],
              max_silent_kept=p["max_sil_kept"], normalize_max=GOLD["normalize_max"], alpha_mix=GOLD["alpha_mix"], sr=p["sr"])
    outs = []
    for k, extra in enumerate((dict(), dict(max_samples=max(len(a) for a in clips)))):
        out = tmp_path / f"out{k}"
        os.makedirs(out)
        data, failed = sl.write_slices(files, out, _load_audio(p["sr"]), **kw, **extra)
        assert data == {n.split(".")[0]: sl.SUCCESS for n in recs if n in GOLD["written"]}
        assert failed == [n.split(".")[0] for n in recs if n in GOLD["failed"]]
        want = {fn: (cnt, digest) for g in recs.values() for fn, cnt, digest in g["files"]}
        assert sorted(os.listdir(out)) == sorted(want)
        for fn, (cnt, digest) in want.items():
            sr, w = wavfile.read(out / fn)
            assert sr == p["sr"] and w.dtype == np.int16 and w.shape == (cnt,), fn
            assert hashlib.sha256(w.tobytes()).hexdigest() == digest, fn
        for g in recs.values():
            for fn, w in g["full"].items():
                assert np.array_equal(wavfile.read(out / fn)[1], w.numpy())
        outs.append({fn: open(out / fn, "rb").read() for fn in want})
    assert outs[0] == outs[1]                                                              # two runs, two batchings: same files


def test_statuses_and_errors_before_device_work(ops, tmp_path):
    from easevoice_trainer_b200 import slicer as sl
    p = GOLD["params"]["default"]
    s = sl.Slicer(**p)
    clips = [so.recording(GOLD["recordings"][n]["spec"], p["sr"]) for n in ("silent.wav", "loud.take2.wav", "short.wav")]
    res = sl.slice_and_normalize(s, clips)
    assert res[0]["status"] == [sl.SLICE_SILENT] and not res[0]["chunks"][0].any()
    assert res[1]["status"] == [sl.SLICE_OK, sl.SLICE_OK] and not res[1]["empty"] and res[2] is None
    before = ops.launches()
    with pytest.raises(ValueError, match="bad.wav"):
        sl.write_slices(["good.wav", "bad.wav"], tmp_path, lambda f, sr: clips[1] if "good" in f else clips[1].reshape(2, -1))
    assert ops.launches() == before and not os.listdir(tmp_path)
