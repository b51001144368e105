"""CPU tests of long-form Whisper transcription: the oracle's seek loop (oracle/whisper_long_oracle.transcribe_long) against the
goldens oracle/pin_asr_long.py pinned against transformers' long-form `generate`, the cases those goldens cover, the seek
rules of `_retrieve_segment` on hand-written hypotheses, and `read_clip` for clips over 30 s."""
import os

import numpy as np
import pytest
import torch

from oracle import pin_asr_long as PINL
from oracle import whisper_long_oracle as L
from oracle import whisper_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "asr_long.pt"), weights_only=False)
SP = O.special_tokens(GOLD["gen"])


def test_oracle_seek_loop_reproduces_goldens():
    """The shorter clip through the float64 seek loop, with its language detected: every window's seek, hypothesis, kept
    tokens and skip flag, and the joined tokens."""
    cfg, sd = GOLD["case"]["cfg"], PINL.make_state_dict(GOLD["case"])
    run = GOLD["runs"][0]
    assert run["language"] is None
    ref = run["results"][1]
    o = L.transcribe_long(sd, cfg, SP, PINL.clip(*GOLD["clips"][1]))
    assert o["language"] == ref["language"] and o["tokens"] == ref["tokens"]
    for w, r in zip(o["windows"], ref["windows"], strict=True):
        assert (w["seek"], w["n_frames"], w["tokens"], w["kept"], w["skipped"]) == \
            (r["seek"], r["n_frames"], r["tokens"], r["kept"], r["skipped"])
        assert abs(w["avg_logprob"] - r["avg_logprob"]) < 1e-9 and abs(w["score"] - r["score"]) < 1e-6


def test_goldens_cover_every_seek_case():
    covered = set()
    for run in GOLD["runs"]:
        for o in run["results"]:
            covered |= PINL.endings(o, SP)
            covered.add("detected" if run["language"] is None else "forced")
    # a single-timestamp ending is not among them: test_retrieve_segment_rules covers that rule
    assert {"pair", "skipped", "short_last", "detected", "forced"} <= covered
    # the forced run keeps its language; every clip is long-form
    assert all(o["language"] == "de" for o in GOLD["runs"][1]["results"])
    assert all(f > 3000 for f in GOLD["frames"])


@pytest.mark.parametrize("impl", ["oracle", "library"])
def test_retrieve_segment_rules(impl):
    if impl == "oracle":
        rs = L.retrieve_segment
    else:
        from easevoice_trainer_b200 import whisper
        rs = whisper.retrieve_segment
    tb = SP["ts_begin"]
    # a pair, then text cut by the window: the tokens up to the pair are kept, seek moves to the pair's first timestamp
    seq = [tb + 0, 5, 6, tb + 40, tb + 40, 7, 8, tb + 90, tb + 91, 9, 10]
    assert rs(seq, tb, 3000) == (seq[:9], 2 * 90)
    # a hypothesis ending in a pair: the same rule
    assert rs(seq[:9], tb, 3000) == (seq[:9], 2 * 90)
    # a single timestamp after text at the end: every token kept, seek moves by the window
    seq2 = [tb + 0, 5, tb + 40, tb + 40, 6, tb + 70]
    assert rs(seq2, tb, 1748) == (seq2, 1748)
    # no pair: everything kept, the whole window
    assert rs([tb + 3, 5, 6, 7], tb, 3000) == ([tb + 3, 5, 6, 7], 3000)
    # no timestamps at all, and an empty hypothesis
    assert rs([5, 6, 7], tb, 2500) == ([5, 6, 7], 2500)
    assert rs([], tb, 3000) == ([], 3000)


def test_read_clip_max_seconds(tmp_path):
    from scipy.io import wavfile

    from easevoice_trainer_b200 import asr
    f = str(tmp_path / "long.wav")
    x = (0.1 * np.sin(np.arange(95 * 16000) * 0.05) * 32767).astype(np.int16)
    wavfile.write(f, 16000, x)
    with pytest.raises(ValueError):
        asr.read_clip(f)
    y, sr = asr.read_clip(f, max_seconds=None)
    assert sr == 16000 and y.size == x.size and y.dtype == np.float32
    f32 = str(tmp_path / "long32.wav")
    wavfile.write(f32, 32000, np.repeat(x, 2))
    assert asr.read_clip(f32, max_seconds=None)[0].size == 2 * x.size
    with pytest.raises(ValueError):
        asr.read_clip(f32, max_seconds=60)


def test_long_pools_fit_the_share():
    from easevoice_trainer_b200 import asr
    n16 = [16000 * s for s in (40, 300, 95, 60, 1200)]
    budget = 300 * 100 * 128 * 4 * 2 / asr.LONG_POOL_SHARE        # two 300 s clips' log-mel fit the share
    pools = asr.long_pools(n16, 128, budget)
    assert [i for p in pools for i in p] == list(range(len(n16)))
    for p in pools:
        T = max(n16[i] for i in p) // 160
        assert len(p) == 1 or len(p) * T * 128 * 4 <= budget * asr.LONG_POOL_SHARE
    assert pools[-1] == [4]                                        # longer than the share alone: a pool of one
