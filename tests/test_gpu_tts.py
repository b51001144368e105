"""GPU tests of the synthesis call (`pytest -m gpu`): evk_fragment_int16 bit for bit against the numpy restatement of
TTS.audio_postprocess (oracle/tts_oracle.py), and ref_spec, prompt_semantic and tts.run end to end against what the
reference's TTS produced with the same seeded models, clips, sentences and vocoder noise (tests/golden/tts.pt,
oracle/pin_tts.py).  The end-to-end tests run in 3xTF32 mode (evk_set_precise(1)), for which the golden's greedy decisions
were chosen to be clear."""
import os
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import tts_oracle as to

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "tts.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
TOL_WAVE = 1e-3


@pytest.fixture(scope="module")
def tts():
    from easevoice_trainer_b200 import lib, tts
    L = lib.init()
    before = L.evk_get_precise()
    L.evk_set_precise(1)
    yield tts
    L.evk_set_precise(before)


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _assemble(tts, audio, bil, split, interval, sr=to.SR):
    dev = [[torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in b] for b in audio]
    return tts.audio_postprocess(dev, sr, bil, 1.0, split, interval)


def test_assembly_synthetic_fragments_bit_identical(tts):
    for (name, audio, bil, split, interval), gold in zip(to.synthetic_fragments(), GOLD["audio_postprocess"]):
        if "raises" in gold:
            with pytest.raises(RuntimeError):
                _assemble(tts, audio, bil, split, interval)
            continue
        sr, out = _assemble(tts, audio, bil, split, interval)
        _, ora = to.audio_postprocess(audio, to.SR, bil, split, interval)
        assert sr == to.SR and out.dtype == np.int16 and np.array_equal(out, ora), name
        assert np.array_equal(out, gold["out"].numpy()), name


def test_assembly_ragged_fragments_bit_identical(tts):
    g = np.random.default_rng(21)
    lens = g.integers(1, 4000, 1000)
    audio, k = [], 0
    while k < len(lens):                                    # buckets of 1 to 8 sentences
        n = int(min(g.integers(1, 9), len(lens) - k))
        audio.append([(np.tanh(g.standard_normal(int(m)) * 3) * g.choice([0.5, 1.0, 1.4])).astype(np.float32)
                      for m in lens[k:k + n]])
        k += n
    audio[3][0][7] = np.nan
    audio[5][0][:] = 0
    audio[7][0][11] = 1.0
    perm = g.permutation(len(lens)).tolist()
    bil, k = [], 0
    for b in audio:
        bil.append(perm[k:k + len(b)])
        k += len(b)
    for split, interval in ((True, 0.3), (False, 0.01)):
        _, out = _assemble(tts, audio, bil, split, interval)
        _, ora = to.audio_postprocess(audio, to.SR, bil, split, interval)
        assert np.array_equal(out, ora), split


def test_assembly_long_fragment_bit_identical(tts):
    g = np.random.default_rng(22)
    a = (np.tanh(g.standard_normal(3_000_001) * 2) * 1.1).astype(np.float32)
    a[2_345_678] = -1.9                                     # the max sits in a late tile
    audio = [[a], [a[:1000].copy()]]
    _, out = _assemble(tts, audio, None, False, 0.3)
    _, ora = to.audio_postprocess(audio, to.SR, None, False, 0.3)
    assert np.array_equal(out, ora)


def test_ref_spec_matches_reference(tts):
    p = GOLD["prompt"]
    clips = to.clips(p["clip_seed"])
    for name, gold in p["specs"].items():
        spec = tts.ref_spec(clips[name][0], 2048, to.SR, 640, 2048, DEV)
        assert spec.shape[0] == 1 and spec.shape[1] == 1025 and spec.shape[2] == gold.shape[2] and spec.dtype == torch.float32
        assert rel(spec[:, ::p["spec_rows"]], gold) < 1e-5, name


def _models():
    from easevoice_trainer_b200 import hubert, models
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    gm, GP = to.gpt_params()
    t2s = Text2SemanticDecoder({"model": gm})
    t2s.load_state_dict(GP)
    sm, SP = to.s2_params()
    vits = models.SynthesizerTrn(1025, 32, n_speakers=300, **sm)
    vits.load_state_dict(SP)
    hm, HP = to.hubert_params()
    hub = hubert.HubertModel({"num_hidden_layers": hm["layers"]})
    hub.load_state_dict(HP)
    return t2s.to(DEV).eval(), vits.to(DEV).eval(), types.SimpleNamespace(model=hub.to(DEV).eval())


def test_prompt_semantic_tokens_identical(tts):
    p = GOLD["prompt"]
    _, vits, hub = _models()
    toks = tts.prompt_semantic(to.clips(p["clip_seed"])["ref.wav"][1], hub, vits, to.SR)
    assert toks.dtype == torch.int64 and toks.cpu().tolist() == p["tokens"].tolist()


class _TTS:
    """The caller's TTS object: the reference's methods around this library's models, the seeded clips as decoded files"""

    def __init__(self, tts, models, n_sent, sent_seed, clip_seed, paths):
        self._tts = tts
        self.t2s_model = types.SimpleNamespace(model=models[0])
        self.vits_model, self.cnhuhbert_model = models[1], models[2]
        self.configs = types.SimpleNamespace(device=DEV, sampling_rate=to.SR, filter_length=2048, hop_length=640, win_length=2048,
                                             hz=to.HZ, max_sec=to.MAX_SEC, languages=to.LANGS, t2s_weights_path="", vits_weights_path="")
        self.text_preprocessor = to.StubPreprocessor(n_sent, sent_seed)
        self.prompt_cache = {"ref_audio_path": None, "prompt_semantic": None, "refer_spec": [], "prompt_text": None,
                             "prompt_lang": None, "phones": None, "bert_features": None, "norm_text": None, "aux_ref_audio_paths": []}
        self.clips = to.clips(clip_seed)
        self.byname = {v: k for k, v in paths.items()}

    def set_ref_audio(self, path):
        self.prompt_cache["prompt_semantic"] = self._tts.prompt_semantic(self.clips[self.byname[path]][1], self.cnhuhbert_model,
                                                                        self.vits_model, self.configs.sampling_rate)
        spec = self._get_ref_spec(path)
        if self.prompt_cache["refer_spec"] in [[], None]:
            self.prompt_cache["refer_spec"] = [spec]
        else:
            self.prompt_cache["refer_spec"][0] = spec
        self.prompt_cache["ref_audio_path"] = path

    def _get_ref_spec(self, path):
        c = self.configs
        return self._tts.ref_spec(self.clips[self.byname[path]][0], c.filter_length, c.sampling_rate, c.hop_length, c.win_length,
                                  c.device)


@pytest.fixture(scope="module")
def models(tts):
    return _models()


@pytest.mark.parametrize("name", list(to.CASES))
def test_run_matches_reference(tts, models, name, monkeypatch):
    gold = GOLD["cases"][name]
    t2s, vits, _ = models
    rec = {"buckets": [], "tokens": []}
    to_batch = tts.to_batch

    def spy_to_batch(*a, **k):
        out = to_batch(*a, **k)
        rec["buckets"].append(out[1])
        return out
    monkeypatch.setattr(tts, "to_batch", spy_to_batch)
    depth = [0]                     # infer_panel_batch_infer hands prompt-free batches to infer_panel_naive_batched
    for meth in ("infer_panel_batch_infer", "infer_panel_naive_batched"):
        orig = getattr(type(t2s), meth).__get__(t2s)

        def spy(*a, _orig=orig, _depth=depth, **k):
            _depth[0] += 1
            try:
                y, idx = _orig(*a, **k)
            finally:
                _depth[0] -= 1
            if _depth[0] == 0:
                rec["tokens"].append(([t.tolist() for t in y], [int(i) for i in idx]))
            return y, idx
        monkeypatch.setattr(t2s, meth, spy, raising=False)
    noise = to.NoiseStream(GOLD["cfg"]["noise_seed"])
    shapes = list(gold["noise_shapes"])
    decode = type(vits).decode.__get__(vits)

    def noisy_decode(codes, text, refer, noise_scale=0.5, speed=1):
        shape = shapes.pop(0)
        return decode(codes, text, refer, noise_scale=noise_scale, speed=speed, noise=noise.draw(shape).to(DEV))
    monkeypatch.setattr(vits, "decode", noisy_decode, raising=False)
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for n in ("ref.wav", "aux.wav"):
            paths[n] = os.path.join(d, n)
            open(paths[n], "wb").close()
        obj = _TTS(tts, models, to.CASES[name]["n_sent"], gold["sent_seed"], gold["clip_seed"], paths)
        inputs = to.case_inputs(name, paths)
        outs = list(tts.run(obj, inputs))
    assert not shapes, "vocoder calls"
    assert rec["buckets"] == gold["buckets"]
    assert rec["tokens"] == [(list(map(list, y)), list(i)) for y, i in gold["tokens"]]
    assert len(outs) == len(gold["outs"])
    gap = int(to.SR * max(inputs["fragment_interval"], 0.01))
    for (sr, out), (gsr, ref), lens in zip(outs, gold["outs"], _fragment_lengths(gold, inputs)):
        ref = ref.numpy()
        assert sr == gsr and out.dtype == np.int16 and out.shape == ref.shape
        zero = np.zeros(ref.shape[0], dtype=bool)
        pos = 0
        for n in lens:
            zero[pos + n:pos + n + gap] = True
            pos += n + gap
        assert pos == ref.shape[0] and not np.any(out[zero]), "silent intervals"
        assert rel(out.astype(np.float64) / 32768, ref.astype(np.float64) / 32768) < TOL_WAVE


def _fragment_lengths(gold, inputs):
    """-> per yield, the sample counts of its fragments in output order: 2 * 640 per token at speed 1 (y[-idx:], where idx 0
    keeps all of y), the vocoder's frames * 640 at other speeds (one call per sentence)"""
    speed = inputs.get("speed_factor", 1.0)
    if speed != 1.0:
        per_call, it = [], iter(gold["noise_shapes"])
        for ys, _ in gold["tokens"]:
            per_call.append([next(it)[-1] * 640 for _ in ys])
    else:
        per_call = [[2 * 640 * len(y[-i:]) for y, i in zip(ys, idx)] for ys, idx in gold["tokens"]]
    if inputs.get("return_fragment"):
        return per_call
    if speed == 1.0 and inputs.get("split_bucket", True):
        return [to.recovery_order(per_call, gold["buckets"][0])]
    return [sum(per_call, [])]
