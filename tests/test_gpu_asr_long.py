"""GPU tests of long-form Whisper transcription (`pytest -m gpu`): the whole-clip log-mel against float64, windows against
today's features and against slices of the whole-clip log-mel, `transcribe_long` against the goldens oracle/pin_asr_long.py
pinned against transformers' long-form `generate`, batch invariance, idle rows, and `WhisperAsr.recognize` on a mix of short
and long wav files."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import pin_asr as PIN
from oracle import pin_asr_long as PINL
from oracle import whisper_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "asr_long.pt"), weights_only=False)
SHORT = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
TOL_MEL = 2e-3            # as test_gpu_asr.test_logmel_against_float64


@pytest.fixture(scope="module")
def W():
    from easevoice_trainer_b200 import lib, whisper
    lib.init().evk_set_precise(0)
    return whisper


def precise(on):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if on else 0)


def batch(xs):
    L = max(x.size for x in xs)
    w = torch.zeros(len(xs), L)
    for i, x in enumerate(xs):
        w[i, :x.size] = torch.from_numpy(x)
    return w.to(DEV), [x.size for x in xs]


def front_end(W, M):
    return W.WhisperModel(dict(W.LARGE_V3, num_mel_bins=M, d_model=128, encoder_attention_heads=2, decoder_attention_heads=2,
                               encoder_layers=1, decoder_layers=1, encoder_ffn_dim=128, decoder_ffn_dim=128,
                               vocab_size=PIN.vocab_size()), SHORT["gen"]).to(DEV)


@pytest.fixture(scope="module")
def net(W):
    c = GOLD["case"]
    m = W.WhisperModel(c["cfg"], GOLD["gen"])
    m.load_state_dict(PINL.make_state_dict(c))
    return m.to(DEV).eval()


def waves():
    return [PINL.clip(*c) for c in GOLD["clips"]]


@pytest.mark.parametrize("M", [80, 128])
def test_logmel_long_against_float64(W, M):
    xs = [PIN.clip(11, 95.3), PIN.clip(7, 0.5), PIN.clip(8, 31.0)]
    xs[0][16000 * 40:16000 * 52] = 0.0                        # a silent stretch: frames at the whole clip's clamp
    m = front_end(W, M)
    w, lens = batch(xs)
    got = m.features_long(w, lens).cpu()
    assert got.shape == (3, xs[0].size // 160, M)
    for i, x in enumerate(xs):
        ref = O.log_mel(x, M)
        T = ref.shape[0]
        err = (got[i, :T].double() - ref).abs().max().item()
        assert err <= TOL_MEL, (i, err)
        assert torch.all(got[i, T:] == 0)


@pytest.mark.parametrize("M", [80, 128])
def test_window_zero_equals_features_for_short_clips(W, M):
    xs = [PIN.clip(101, 4.37), PIN.clip(102, 29.99), PIN.clip(103, 30.0)]
    m = front_end(W, M)
    w, lens = batch(xs)
    f = m.features(w, lens)
    lm = m.features_long(w, lens)
    tab = torch.tensor([[i, 0, n // 160] for i, n in enumerate(lens)], dtype=torch.int32, device=DEV)
    from easevoice_trainer_b200 import ops
    assert torch.equal(ops.whisper_window(lm, tab), f)


def test_window_equals_sliced_log_mel(W):
    from easevoice_trainer_b200 import ops
    m = front_end(W, 128)
    xs = [PIN.clip(12, 95.0), PIN.clip(13, 41.3)]
    w, lens = batch(xs)
    lm = m.features_long(w, lens)
    rows = [(0, 0, 3000), (0, 1234, 3000), (1, 2968, 4130 - 2968), (0, 9400, 100), (1, 0, 0)]
    out = ops.whisper_window(lm, torch.tensor(rows, dtype=torch.int32, device=DEV))
    for r, (c, s, n) in enumerate(rows):
        ref = torch.zeros(3000, 128, device=DEV)
        ref[:n] = lm[c, s:s + n]
        assert torch.equal(out[r], ref), r


def oracle_lm(xs, M):
    lms = [O.log_mel(x, M) for x in xs]
    out = torch.zeros(len(lms), max(lm.shape[0] for lm in lms), M)
    for i, lm in enumerate(lms):
        out[i, :lm.shape[0]] = lm.float()
    return out.to(DEV), [lm.shape[0] for lm in lms]


def test_transcribe_long_against_goldens(W, net):
    """Under 3xTF32, on the oracle's whole-clip features: the two clips as one pool, with detection and with a forced
    language: tokens, seeks, hypotheses, skip flags and languages equal the goldens; scores within the short-form bound."""
    precise(True)
    try:
        lm, frames = oracle_lm(waves(), net.cfg["num_mel_bins"])
        assert frames == GOLD["frames"]
        for run in GOLD["runs"]:
            got = net.transcribe_long(lm, frames, language=run["language"], clips_per_batch=2)
            for i, (o, r) in enumerate(zip(got, run["results"], strict=True)):
                assert o["language"] == r["language"] and o["tokens"] == r["tokens"], (i, run["language"])
                assert len(o["windows"]) == len(r["windows"])
                for w, rw in zip(o["windows"], r["windows"]):
                    assert (w["seek"], w["n_frames"], w["tokens"], w["kept"], w["skipped"]) == \
                        (rw["seek"], rw["n_frames"], rw["tokens"], rw["kept"], rw["skipped"]), (i, rw["seek"])
                    for k in ("score", "avg_logprob"):
                        assert abs(w[k] - rw[k]) <= 1e-4 * max(1.0, abs(rw[k])), (i, k, w[k], rw[k])
                    assert abs(w["no_speech_prob"] - rw["no_speech_prob"]) <= 1e-4 * rw["no_speech_prob"] + 1e-7
    finally:
        precise(False)


def test_batch_invariance_and_idle_rows(W, net):
    """A clip gives the same log-mel bits, tokens and seeks alone and inside a pool; a round whose other row has no window
    left takes no more decode steps than the clip alone; one row round-robin over the pool gives the same results."""
    xs = waves()
    w, lens = batch(xs)
    lm2 = net.features_long(w, lens)
    w1, l1 = batch(xs[:1])
    lm1 = net.features_long(w1, l1)
    frames = [n // 160 for n in lens]
    assert torch.equal(lm2[0, :frames[0]], lm1[0])
    precise(True)
    try:
        alone = net.transcribe_long(lm1, frames[:1], language="de", clips_per_batch=1)[0]
        pool = net.transcribe_long(lm2, frames, language="de", clips_per_batch=2)
        rr = net.transcribe_long(lm2, frames, language="de", clips_per_batch=1)
    finally:
        precise(False)
    assert pool[0]["tokens"] == alone["tokens"]
    assert [w["seek"] for w in pool[0]["windows"]] == [w["seek"] for w in alone["windows"]]
    # the goldens' first clip has more windows than the second: its last round has an idle row
    gold = GOLD["runs"][1]["results"]
    n_other = len(gold[1]["windows"])
    assert len(gold[0]["windows"]) > n_other and len(pool[1]["windows"]) == n_other
    for wp, wa in zip(pool[0]["windows"][n_other:], alone["windows"][n_other:], strict=True):
        assert wp["steps"] <= wa["steps"], (wp["steps"], wa["steps"])
    assert [o["tokens"] for o in rr] == [o["tokens"] for o in pool]


def tokenizer(mdir, n_text):
    from tokenizers import Tokenizer, models
    vocab = {f"w{i}": i for i in range(n_text)}
    vocab["[UNK]"] = n_text
    Tokenizer(models.WordLevel(vocab=vocab, unk_token="[UNK]")).save(str(mdir / "tokenizer.json"))
    return Tokenizer.from_file(str(mdir / "tokenizer.json"))


def test_recognize_short_and_long(W, tmp_path):
    from scipy.io import wavfile

    from easevoice_trainer_b200 import asr
    c = GOLD["case"]
    mdir = tmp_path / "model"
    mdir.mkdir()
    json.dump(dict(c["cfg"]), open(mdir / "config.json", "w"))
    json.dump(GOLD["gen"], open(mdir / "generation_config.json", "w"))
    torch.save(PINL.make_state_dict(c), mdir / "pytorch_model.bin")
    tok = tokenizer(mdir, GOLD["n_text"])
    files = {}
    for name, x in (("s0", PIN.clip(50, 3.1)), ("l0", waves()[0]), ("s1", PIN.clip(51, 7.45)), ("l1", waves()[1])):
        files[name] = str(tmp_path / f"{name}.wav")
        wavfile.write(files[name], 16000, x.astype(np.float32))
    a = asr.WhisperAsr("large-v3", "auto", "float32", model_dir=str(mdir))
    precise(True)
    try:
        mixed = [files[k] for k in ("s0", "l0", "s1", "l1")]
        res = a.recognize(mixed, str(tmp_path / "mixed.list"), str(tmp_path / "mixed.dump"))
        assert res.status == "success", res.message
        lines = open(tmp_path / "mixed.list", encoding="utf-8").read().split("\n")
        res_s = a.recognize([files["s0"], files["s1"]], str(tmp_path / "short.list"), str(tmp_path / "short.dump"))
        short_lines = open(tmp_path / "short.list", encoding="utf-8").read().split("\n")
    finally:
        precise(False)
    assert [ln.split("|", 1)[0] for ln in lines] == mixed
    assert [lines[0], lines[2]] == short_lines
    for f in (files["s0"], files["s1"]):
        assert res.data[f] == res_s.data[f] and "windows" not in res.data[f]
    for k, r in zip(("l0", "l1"), GOLD["runs"][0]["results"]):
        f = files[k]
        line = lines[mixed.index(f)]
        assert line == f"{f}|{r['language']}|{tok.decode([t for t in r['tokens'] if t < GOLD['n_text']])}"
        info = res.data[f]
        assert len(info["windows"]) == len(r["windows"])
        assert [w["skipped"] for w in info["windows"]] == [w["skipped"] for w in r["windows"]]
        assert info["windows"][0]["start_s"] == 0.0 and info["no_speech_prob"] == info["windows"][0]["no_speech_prob"]
        assert set(info) >= {"status", "avg_logprob", "compression_ratio", "no_speech_prob"}
