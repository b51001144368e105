"""CPU tests of tts.run_many's host side: request checks and error isolation, each request's buckets against to_batch of
that request alone, the decoding calls and their packing into decoder batches of at most 64 rows, the per-row tables of
Text2SemanticDecoder.decode_groups and the noise seeds a request's decoding calls draw after set_seed."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import tts_oracle as to

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def tts():
    from easevoice_trainer_b200 import tts
    return tts


class _HostTTS:
    """A caller's TTS object on the CPU: set_ref_audio / _get_ref_spec record their calls and store small tensors"""

    def __init__(self, n_sent=5, seed=3):
        self.configs = types.SimpleNamespace(languages=to.LANGS, sampling_rate=32000, device=torch.device("cpu"), hz=50,
                                             max_sec=6)
        self.prompt_cache = {"ref_audio_path": None, "prompt_semantic": None, "refer_spec": [], "prompt_text": None,
                             "prompt_lang": None, "phones": None, "bert_features": None, "norm_text": None,
                             "aux_ref_audio_paths": []}
        self.text_preprocessor = to.StubPreprocessor(n_sent, seed)
        self.t2s_model = types.SimpleNamespace(model=types.SimpleNamespace(vocab_size=1025))
        self.calls = []

    def set_ref_audio(self, path):
        self.calls.append(("ref", path))
        if "short" in path:
            raise OSError("audio length should be in 3~10 seconds.")
        self.prompt_cache["prompt_semantic"] = torch.full((7,), len(path), dtype=torch.int64)
        spec = torch.full((1, 3, 2), float(len(path)))
        if self.prompt_cache["refer_spec"] in [[], None]:
            self.prompt_cache["refer_spec"] = [spec]
        else:
            self.prompt_cache["refer_spec"][0] = spec
        self.prompt_cache["ref_audio_path"] = path

    def _get_ref_spec(self, path):
        self.calls.append(("aux", path))
        return torch.zeros(1, 3, 2)


@pytest.fixture()
def clips(tmp_path):
    out = {}
    for n in ("a.wav", "bb.wav", "short.wav", "aux.wav"):
        out[n] = str(tmp_path / n)
        open(out[n], "wb").close()
    return out


def _req(path, **kw):
    return dict(dict(text="t", text_lang="zh", prompt_text="p", prompt_lang="zh", ref_audio_path=path, batch_size=2, seed=5), **kw)


def test_return_fragment_raises_before_any_work(tts):
    t = _HostTTS()
    with pytest.raises(ValueError, match="return_fragment"):
        tts.run_many(t, [_req("x.wav"), _req("y.wav", return_fragment=True)])
    assert t.calls == [] and t.prompt_cache["ref_audio_path"] is None


def test_rejected_requests_get_zeros_and_an_error_entry(tts, clips):
    t = _HostTTS()
    bad = [_req(os.path.join(ROOT, "no", "such.wav")), _req(clips["a.wav"], text_lang="xx"), _req(""),
           _req(clips["short.wav"]), _req(clips["a.wav"], top_k=0)]
    results, errors = tts.run_many(t, bad)
    assert [i for i, _ in errors] == [0, 1, 2, 3, 4]
    assert [type(e) for _, e in errors] == [ValueError, AssertionError, ValueError, OSError, ValueError]
    for sr, a in results:
        assert sr == 32000 and a.dtype == np.int16 and a.shape == (32000,) and not a.any()


def test_requests_share_clip_reads_and_leave_the_cache_as_run(tts, clips):
    t = _HostTTS()
    reqs = [_req(clips["a.wav"]), _req(clips["bb.wav"], aux_ref_audio_paths=[clips["aux.wav"]]), _req(clips["short.wav"]),
            _req(clips["a.wav"], prompt_text="q"), _req(clips["bb.wav"], aux_ref_audio_paths=[clips["aux.wav"]])]
    memo = {"ref": {}, "aux": {}, "prompt": {}}
    states = []
    for r in reqs:
        try:
            states.append(tts._request(t, r, memo))
        except OSError:
            states.append(None)
    # each distinct clip read once, the failing one included; the aux clip once
    assert t.calls == [("ref", clips["a.wav"]), ("ref", clips["bb.wav"]), ("aux", clips["aux.wav"]), ("ref", clips["short.wav"])]
    assert states[2] is None
    assert states[0]["prompt"].tolist() == [len(clips["a.wav"])] * 7 and len(states[0]["refer"]) == 1
    assert states[1]["prompt"].tolist() == [len(clips["bb.wav"])] * 7 and len(states[1]["refer"]) == 2
    assert states[3]["prompt"].tolist() == [len(clips["a.wav"])] * 7 and len(states[3]["refer"]) == 1
    c = t.prompt_cache
    assert c["ref_audio_path"] == clips["bb.wav"] and c["aux_ref_audio_paths"] == [clips["aux.wav"]]
    assert len(c["refer_spec"]) == 2 and c["prompt_text"] == "p。"


def test_buckets_equal_to_batch_of_the_request_alone(tts, clips):
    t = _HostTTS(n_sent=9, seed=4)
    memo = {"ref": {}, "aux": {}, "prompt": {}}
    for bs, split in ((1, True), (3, True), (4, False)):
        st = tts._request(t, _req(clips["a.wav"], batch_size=bs, split_bucket=split), memo)
        data = t.text_preprocessor.preprocess("t", "zh", "cut0")
        alone, bil = tts.to_batch(data, t.prompt_cache, bs, 0.75, split, torch.device("cpu"))
        assert st["bil"] == bil
        for a, b in zip(st["batches"], alone):
            assert [x.tolist() for x in a["all_phones"]] == [x.tolist() for x in b["all_phones"]] and a["max_len"] == b["max_len"]


def test_decoding_calls_and_packing(tts):
    item = lambda n: {"all_phones": [None] * n}                 # noqa: E731
    batches = [item(3), item(1), item(130)]
    assert tts.decode_units(batches, False, True) == [(0, [0, 1, 2], 1, False), (1, [0], 1, False),
                                                      (2, list(range(64)), 1, False), (2, list(range(64, 128)), 1, False),
                                                      (2, [128, 129], 1, False)]
    assert tts.decode_units(batches[:2], False, False) == [(0, [0], 11, True), (0, [1], 11, True), (0, [2], 11, True),
                                                           (1, [0], 11, True)]
    assert tts.decode_units(batches[:2], True, True) == [(0, [0, 1, 2], 11, False), (1, [0], 11, False)]
    sizes = [3, 64, 1, 60, 2, 2, 30, 34, 1]
    packs = tts.pack_units(sizes)
    assert packs == [[0], [1], [2, 3, 4], [5, 6], [7, 8]]
    assert sum(packs, []) == list(range(len(sizes))) and all(sum(sizes[i] for i in p) <= 64 for p in packs)


def test_row_tables(tts):
    from easevoice_trainer_b200.models_gpt import row_tables
    g = lambda n, ml, yp, **kw: dict(dict(rows=[None] * n, lens=list(range(3, 3 + n)), max_len=ml,  # noqa: E731
                                          prompt=None if yp is None else torch.zeros(yp), top_k=5, top_p=0.9,
                                          temperature=0.7, repetition_penalty=1.2, early_stop_num=300, eos_steps=1), **kw)
    groups = [g(2, 10, 40), g(1, 20, None, eos_steps=11, top_k=1), g(3, 12, 45, top_p=1.0)]
    icfg, fcfg, skip, pref = row_tables(groups, 1500)
    L0 = 57
    assert icfg == [[0, 40, L0, 5, 300, 1500, 1, 0], [0, 40, L0, 5, 300, 1500, 1, 1], [0, 0, L0, 1, 300, 1500, 11, 0],
                    [0, 45, L0, 5, 300, 1500, 1, 0], [0, 45, L0, 5, 300, 1500, 1, 1], [0, 45, L0, 5, 300, 1500, 1, 2]]
    assert fcfg[0] == [0.9, pytest.approx(0.7), pytest.approx(1.2), 0.0] and fcfg[3][0] == 1.0
    assert skip == [[3, 17], [4, 17], [3, 57], [3, 12], [4, 12], [5, 12]]
    assert pref == [40, 40, 0, 45, 45, 45]


def test_unit_seeds_are_the_draws_after_set_seed(tts):
    tts.set_seed(77)
    seeds = tts.unit_seeds(3, torch.device("cpu"))
    torch.manual_seed(77)
    ref = [int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64)) for _ in range(3)]
    assert seeds.tolist() == ref and len(set(ref)) == 3
