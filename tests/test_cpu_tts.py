"""CPU tests of the synthesis call (easevoice-trainer_b200/tts.py): bucketing against the reference's `TTS.to_batch`, the
numpy restatement of `TTS.audio_postprocess` against the reference's output (tests/golden/tts.pt, oracle/pin_tts.py), and
the argument errors that must come before any device work."""
import os

import numpy as np
import pytest
import torch

from oracle import tts_oracle as to

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "tts.pt"), weights_only=False)


@pytest.fixture(scope="module")
def tts():
    from easevoice_trainer_b200 import tts
    return tts


def test_to_batch_buckets_match_reference(tts):
    cases = to.bucket_cases()
    assert len(cases) == len(GOLD["buckets"])
    for (lens, bs, th), gold in zip(cases, GOLD["buckets"]):
        data = [{"norm_text": "t" * n, "phones": [1, 2], "bert_features": torch.zeros(1024, 2)} for n in lens]
        batches, bil = tts.to_batch(data, None, bs, th, True, torch.device("cpu"))
        assert bil == gold, (lens, bs, th)
        assert [b["norm_text"] for b in batches] == [["t" * lens[i] for i in b] for b in bil]
        assert tts.recovery_order([[(i, j) for j in range(len(b))] for i, b in enumerate(bil)], bil) == \
            [next((i, j) for i, b in enumerate(bil) for j, k in enumerate(b) if k == s) for s in range(len(lens))]


def test_to_batch_with_prompt_and_without_buckets(tts):
    sent = to.sentences(5, 3)
    prompt = to.sentences(1, 4)[0]
    batches, bil = tts.to_batch(sent, prompt, 2, 0.75, False, torch.device("cpu"))
    assert bil == [[0, 1], [2, 3], [4]]
    b = batches[1]
    assert [p.tolist() for p in b["phones"]] == [sent[2]["phones"], sent[3]["phones"]]
    assert [p.tolist() for p in b["all_phones"]] == [prompt["phones"] + sent[i]["phones"] for i in (2, 3)]
    assert b["all_phones_len"].tolist() == [len(prompt["phones"]) + len(sent[i]["phones"]) for i in (2, 3)]
    assert torch.equal(b["all_bert_features"][0], torch.cat([prompt["bert_features"], sent[2]["bert_features"]], 1))
    assert b["max_len"] == max(len(prompt["phones"]) + len(sent[i]["phones"]) for i in (2, 3))


def test_oracle_audio_postprocess_matches_reference():
    for (name, audio, bil, split, interval), gold in zip(to.synthetic_fragments(), GOLD["audio_postprocess"]):
        assert gold["name"] == name
        if "raises" in gold:
            with pytest.raises(ValueError):
                to.audio_postprocess(audio, to.SR, bil, split, interval)
            continue
        sr, out = to.audio_postprocess(audio, to.SR, bil, split, interval)
        assert sr == to.SR and out.dtype == np.int16
        assert np.array_equal(out, gold["out"].numpy()), name


def test_saturated_sample_wraps_like_the_reference():
    _, out = to.audio_postprocess([[np.array([1.0, -1.0, 0.5], np.float32)]], 100, None, False, 0.02)
    assert out.tolist() == [-32768, -32768, 16384, 0, 0]


def test_prompt_semantic_rejects_clip_length_before_device_work(tts):
    for n in (47999, 160001, 0):
        with pytest.raises(OSError, match="3~10 seconds"):
            tts.prompt_semantic(np.zeros(n, np.float32), None, None, 32000)


class _Cfg:
    languages = to.LANGS
    sampling_rate = 32000
    device = "cpu"


class _NoDeviceTTS:
    """a TTS whose every model access fails: the checks of run must come first"""
    configs = _Cfg()
    prompt_cache = {"ref_audio_path": None, "prompt_semantic": None, "refer_spec": [], "prompt_text": None,
                    "aux_ref_audio_paths": []}
    t2s_model = type("T2S", (), {"model": type("M", (), {"infer_panel_batch_infer": None, "infer_panel_naive_batched": None})()})()

    def set_ref_audio(self, path):
        raise AssertionError("set_ref_audio must not run")


def test_run_rejects_missing_reference_before_device_work(tts):
    with pytest.raises(ValueError, match="ref_audio_path cannot be empty"):
        next(tts.run(_NoDeviceTTS(), {"text": "x", "text_lang": "zh", "ref_audio_path": ""}))
    with pytest.raises(ValueError, match="not exists"):
        next(tts.run(_NoDeviceTTS(), {"text": "x", "text_lang": "zh", "ref_audio_path": os.path.join(ROOT, "no", "such.wav")}))
    with pytest.raises(AssertionError):
        next(tts.run(_NoDeviceTTS(), {"text": "x", "text_lang": "xx", "ref_audio_path": "a.wav"}))
