"""CPU tests of Whisper transcription: the oracle (oracle/whisper_oracle.py) against the goldens oracle/pin_asr.py pinned
against transformers, where the feature-domain padding differs from the extractor's waveform padding, and the host logic of
`WhisperAsr` (validation, the FAILED path, the list format, text decoding, the no-speech rule, batch sizing)."""
import os

import numpy as np
import pytest
import torch

from oracle import pin_asr as PIN
from oracle import whisper_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "asr.pt"), weights_only=False)


@pytest.fixture(scope="module")
def A():
    from easevoice_trainer_b200 import asr
    return asr


@pytest.mark.parametrize("M", [80, 128])
def test_feature_padding_differs_only_at_the_tail(M):
    """Frames of the clip away from its end equal the extractor's; from the last frames on they differ: the extractor pads
    the waveform to 30 s (its frames there are log-mel of silence clamped at the max - 8, and its last frames see zeros
    instead of the reflection), the library pads the normalised features with zeros."""
    fe = GOLD["frontend"][M]
    ours = O.features(PIN.clip(fe["seed"], fe["secs"]), M)
    T, hf = fe["n_frames"], fe["hf_head"].double()
    assert (ours[:T - 3] - hf[:T - 3]).abs().max() < 1e-5
    assert torch.all(ours[T:] == 0)
    assert (hf[T + 8:T + 16] - hf[T + 8]).abs().max() == 0 and hf[T + 8].abs().min() > 0.1
    assert torch.all(fe["hf_last"] == hf[T + 8].float())


def test_filters_match_library(A):
    from easevoice_trainer_b200 import whisper
    for M in (80, 128):
        assert np.array_equal(whisper.mel_filters(M), O.mel_filters(M))


def test_processors_against_goldens():
    sp = O.special_tokens(GOLD["gen"])
    for c in GOLD["processors"]:
        got = O.process(c["lp"], c["hists"], sp)
        assert torch.equal(got, c["out"])


def test_oracle_beam_search_against_generate_goldens():
    sp = O.special_tokens(GOLD["gen"])
    c = GOLD["cases"]["m80_d2"]
    sd = PIN.make_state_dict(c["cfg"], c["seed"], c["eot_gain"])
    feats = O.features(PIN.clip(c["seed"] * 10, c["secs"][0]), c["cfg"]["num_mel_bins"])
    for run in c["runs"]:
        o = O.transcribe_clip(sd, c["cfg"], sp, feats, language=run["language"])
        assert o["tokens"] == run["results"][0]["tokens"] and o["language"] == run["results"][0]["language"]


def test_special_tokens_from_generation_config(A):
    from easevoice_trainer_b200 import whisper
    sp = whisper.special_tokens(GOLD["gen"])
    assert sp == O.special_tokens(GOLD["gen"])
    with pytest.raises(ValueError):
        whisper.WhisperModel(dict(GOLD["cases"]["m80_d2"]["cfg"], vocab_size=1500), GOLD["gen"])
    with pytest.raises(ValueError):
        whisper.WhisperModel(dict(GOLD["cases"]["m80_d2"]["cfg"], d_model=96), GOLD["gen"])


def test_strict_loading(A):
    from easevoice_trainer_b200 import whisper
    c = GOLD["cases"]["m80_d2"]
    net = whisper.WhisperModel(c["cfg"], GOLD["gen"])
    sd = PIN.make_state_dict(c["cfg"], c["seed"])
    net.load_state_dict(dict(sd, **{"proj_out.weight": sd["model.decoder.embed_tokens.weight"]}))
    for bad in ({k: v for k, v in sd.items() if k != "model.decoder.layer_norm.bias"}, dict(sd, extra=torch.zeros(1)),
                dict(sd, **{"model.encoder.conv1.bias": torch.zeros(3)})):
        with pytest.raises(ValueError):
            net.load_state_dict(bad)


def test_validation_and_failed_path(A, tmp_path, monkeypatch):
    from scipy.io import wavfile
    with pytest.raises(ValueError):
        A.WhisperAsr("huge", "zh", "float16")
    with pytest.raises(ValueError):
        A.WhisperAsr("large-v3", "xx", "float16")
    ok = str(tmp_path / "ok.wav")
    wavfile.write(ok, 32000, np.zeros(32000, dtype=np.int16))
    bad_sr = str(tmp_path / "sr.wav")
    wavfile.write(bad_sr, 22050, np.zeros(22050, dtype=np.int16))
    long = str(tmp_path / "long.wav")
    wavfile.write(long, 16000, np.zeros(16000 * 31, dtype=np.int16))
    missing = str(tmp_path / "missing.wav")
    int32 = str(tmp_path / "int32.wav")
    wavfile.write(int32, 16000, np.zeros(16000, dtype=np.int32))
    for f in (bad_sr, long, missing, int32):
        with pytest.raises(Exception):
            A.read_clip(f)
    a = A.WhisperAsr("large-v3", "auto", "float16")
    monkeypatch.setattr(a, "load", lambda: (None, None))
    out = tmp_path / "asr.list"
    res = a.recognize([ok, bad_sr, long], str(out), str(tmp_path / "dump"))
    assert res.status == "failed" and res.data == {ok: "success", bad_sr: "failed"} and not out.exists()
    class M:
        sp = dict(langs={"en": 1})
    yue = A.WhisperAsr("large-v2", "yue", "float16")
    monkeypatch.setattr(yue, "load", lambda: (M, None))
    res = yue.recognize([ok], str(out), str(tmp_path / "dump"))
    assert res.status == "failed" and "yue" in res.message and not out.exists()
    monkeypatch.setattr(a, "load", lambda: (_ for _ in ()).throw(OSError("no model")))
    assert a.recognize([ok], str(out), str(tmp_path / "dump")).message == "Failed to load model"


def test_text_and_rules(A, tmp_path):
    from tokenizers import Tokenizer, models
    t = Tokenizer(models.WordLevel(vocab={"a": 0, "b": 1, "[UNK]": 2}, unk_token="[UNK]"))
    assert A.decode_text(t, [0, 1, 0, 5, 7], eot=2) == t.decode([0, 1, 0])
    assert A.is_no_speech(0.7, -1.5) and not A.is_no_speech(0.7, -0.5) and not A.is_no_speech(0.5, -2.0)
    assert A.compression_ratio("") == 0.0 and A.compression_ratio("ab" * 100) > 2
    from easevoice_trainer_b200 import whisper
    assert A.clips_per_batch(whisper.LARGE_V3) == 14
