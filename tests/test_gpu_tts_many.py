"""GPU tests of tts.run_many (`pytest -m gpu`) on the seeded small models of test_gpu_tts.py: every request's semantic
tokens against its own tts.run, the first logits of ragged-prompt rows against the row decoded alone
(Text2SemanticDecoder.decode_groups), a request's audio against the same request in a larger call, the reference golden
(tests/golden/tts.pt) with the golden's vocoder noise, and the rejects.  3xTF32 mode throughout, as in test_gpu_tts.py."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import tts_oracle as to
from tests.test_gpu_tts import DEV, GOLD, TOL_WAVE, _TTS, _fragment_lengths, _models, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tts():
    from easevoice_trainer_b200 import lib, tts
    L = lib.init()
    before = L.evk_get_precise()
    L.evk_set_precise(1)
    yield tts
    L.evk_set_precise(before)


@pytest.fixture(scope="module")
def models(tts):
    return _models()


def _clip(seed, seconds):
    g = torch.Generator().manual_seed(seed)
    n = int(32000 * seconds)
    t = torch.arange(n) / 32000.0
    x = (0.4 * torch.sin(2 * np.pi * (110 + 90 * torch.rand(1, generator=g)) * t) + 0.05 * torch.randn(n, generator=g)).float()
    return x.numpy(), x[::2].contiguous().numpy()


class _Caller(_TTS):
    """_TTS with clips of several lengths (prompts of different lengths) and a record of the vocoder's code sequences"""

    def __init__(self, tts, models, paths, clips, n_sent=5, sent_seed=8):
        super().__init__(tts, models, n_sent, sent_seed, 0, paths)
        self.clips = clips
        self.codes = []
        decode = type(self.vits_model).decode.__get__(self.vits_model)

        decode_batch = type(self.vits_model).decode_batch.__get__(self.vits_model)

        def spy(codes, text, refer, noise_scale=0.5, speed=1, noise=None):
            self.codes.append(codes.reshape(-1).tolist())
            return decode(codes, text, refer, noise_scale=noise_scale, speed=speed, noise=noise)

        def spy_batch(codes_list, *a, **k):
            self.codes += [c.tolist() for c in codes_list]
            return decode_batch(codes_list, *a, **k)
        self.vits_model.decode = spy
        self.vits_model.decode_batch = spy_batch


@pytest.fixture()
def files():
    with tempfile.TemporaryDirectory() as d:
        clips = {f"c{i}.wav": _clip(40 + i, s) for i, s in enumerate((3.2, 4.5, 6.1, 8.0, 3.6))}
        paths = {}
        for n in clips:
            paths[n] = os.path.join(d, n)
            open(paths[n], "wb").close()
        yield paths, clips


REQS = [dict(top_k=1, top_p=1, temperature=1, repetition_penalty=1.35, seed=3, batch_size=2),
        dict(top_k=15, top_p=0.8, temperature=0.9, repetition_penalty=1.2, seed=11, batch_size=3),
        dict(top_k=5, top_p=1, temperature=1.3, repetition_penalty=1.0, seed=7, batch_size=1),
        dict(top_k=30, top_p=0.6, temperature=0.7, repetition_penalty=1.5, seed=19, batch_size=2, parallel_infer=False),
        dict(top_k=3, top_p=0.95, temperature=1, repetition_penalty=1.35, seed=23, batch_size=4, speed_factor=1.25)]


def _inputs(paths, i, **kw):
    return dict(dict(text="t", text_lang="zh", prompt_text="prompt", prompt_lang="zh", ref_audio_path=paths[f"c{i}.wav"],
                     fragment_interval=0.05), **REQS[i], **kw)


def test_tokens_equal_each_requests_own_run(tts, models, files):
    paths, clips = files
    obj = _Caller(tts, models, paths, clips)
    solo = []
    for i in range(len(REQS)):
        obj.codes.clear()
        list(tts.run(obj, _inputs(paths, i)))
        solo.append(list(obj.codes))
    obj.codes.clear()
    results, errors = tts.run_many(obj, [_inputs(paths, i) for i in range(len(REQS))])
    assert errors == [] and len(results) == len(REQS)
    # run_many vocodes the speed-1 buckets of all requests together after the per-sentence calls: the same code sequences
    assert sorted(obj.codes) == sorted(sum(solo, []))
    assert any(len(set(c)) > 1 for c in obj.codes)


def test_ragged_prompt_rows_first_logits_bit_identical(tts, models):
    t2s = models[0]
    sent = to.sentences(4, 31)
    g = torch.Generator().manual_seed(5)
    groups = []
    for k, yp in enumerate((37, 12, 60, 25)):
        row = torch.tensor(sent[k]["phones"], device=DEV)
        groups.append(dict(rows=[row], lens=[row.shape[0]], bert=[sent[k]["bert_features"].to(DEV)], max_len=row.shape[0] + k,
                           prompt=torch.randint(0, 1024, (yp,), generator=g).to(DEV), seed=torch.tensor([k], device=DEV),
                           eos_steps=1, top_k=1, top_p=1.0, temperature=1.0, repetition_penalty=1.35, early_stop_num=40))
    trace = []
    ys, _ = t2s.decode_groups(groups, trace=trace)
    for b, gr in enumerate(groups):
        alone = []
        y1, _ = t2s.infer_panel_batch_infer(gr["rows"], torch.tensor(gr["lens"]), gr["prompt"][None], gr["bert"], top_k=1,
                                            early_stop_num=40, max_len=gr["max_len"], trace=alone)
        assert torch.equal(trace[0][b], alone[0][0]), b
        assert torch.equal(ys[b], y1[0]), b


def _solo_many(tts, obj, inputs):
    obj.codes.clear()
    (res,), errors = tts.run_many(obj, [inputs])
    assert errors == []
    return res, list(obj.codes)


def test_request_alone_and_among_others(tts, models, files):
    paths, clips = files
    obj = _Caller(tts, models, paths, clips)
    r = _inputs(paths, 1)
    (sr, alone), codes = _solo_many(tts, obj, r)
    obj.codes.clear()
    results, errors = tts.run_many(obj, [r, _inputs(paths, 0), _inputs(paths, 2), _inputs(paths, 3)])
    assert errors == [] and results[0][0] == sr
    assert all(c in obj.codes for c in codes)
    assert results[0][1].shape == alone.shape
    assert rel(results[0][1].astype(np.float64), alone.astype(np.float64)) < TOL_WAVE


@pytest.mark.parametrize("name", [n for n in to.CASES if not to.CASES[n]["inputs"].get("return_fragment")])
def test_run_many_matches_reference_golden(tts, models, name):
    gold = GOLD["cases"][name]
    noise = to.NoiseStream(GOLD["cfg"]["noise_seed"])
    shapes = list(gold["noise_shapes"])

    def draw(i, c, shape):
        s = shapes.pop(0)
        assert tuple(s) == (1, shape[2], shape[1])
        return noise.draw(s).to(DEV).transpose(1, 2).contiguous()
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for n in ("ref.wav", "aux.wav"):
            paths[n] = os.path.join(d, n)
            open(paths[n], "wb").close()
        obj = _TTS(tts, models, to.CASES[name]["n_sent"], gold["sent_seed"], gold["clip_seed"], paths)
        inputs = to.case_inputs(name, paths)
        ((sr, out),), errors = tts.run_many(obj, [inputs], noise=draw)
    assert errors == [] and not shapes
    (gsr, ref), = gold["outs"]
    ref = ref.numpy()
    assert sr == gsr and out.dtype == np.int16 and out.shape == ref.shape
    gap = int(to.SR * max(inputs["fragment_interval"], 0.01))
    zero, pos = np.zeros(ref.shape[0], dtype=bool), 0
    for n in _fragment_lengths(gold, inputs)[0]:
        zero[pos + n:pos + n + gap] = True
        pos += n + gap
    assert not np.any(out[zero])
    assert rel(out.astype(np.float64) / 32768, ref.astype(np.float64) / 32768) < TOL_WAVE


def test_rejects_leave_the_other_requests_alone(tts, models, files):
    paths, clips = files
    obj = _Caller(tts, models, paths, clips)
    with pytest.raises(ValueError, match="return_fragment"):
        tts.run_many(obj, [_inputs(paths, 0), _inputs(paths, 2, return_fragment=True)])
    good = [_inputs(paths, 0), _inputs(paths, 2)]
    ref, errors = tts.run_many(obj, good)
    assert errors == []
    bad = dict(good[0], ref_audio_path=os.path.join(os.path.dirname(paths["c0.wav"]), "missing.wav"))
    out, errors = tts.run_many(obj, [good[0], bad, good[1]])
    assert [i for i, _ in errors] == [1] and isinstance(errors[0][1], ValueError)
    assert out[1][1].shape == (to.SR,) and not out[1][1].any()
    for a, b in zip((out[0], out[2]), ref):
        assert a[0] == b[0] and a[1].shape == b[1].shape
        assert rel(a[1].astype(np.float64), b[1].astype(np.float64)) < TOL_WAVE


def test_decode_batch_rows_match_decode_alone(tts, models):
    vits = models[1]
    g = torch.Generator().manual_seed(17)
    T = [23, 61, 9, 40]
    codes = [torch.randint(0, 1024, (t,), generator=g).to(DEV) for t in T]
    text = [torch.randint(0, 732, (x,), generator=g).to(DEV) for x in (11, 30, 5, 19)]
    refers = [[tts.ref_spec(_clip(60 + b, 3.0 + b)[0], 2048, to.SR, 640, 2048, DEV)] for b in range(len(T))]
    refers[1].append(tts.ref_spec(_clip(70, 4.2)[0], 2048, to.SR, 640, 2048, DEV))         # a row with an aux clip
    ge = torch.cat([vits.ref_style(r) for r in refers])
    noise = [torch.randn(2 * t, 192, generator=g).to(DEV) for t in T]
    batch = vits.decode_batch(codes, text, ge, noise=noise)
    for b in range(len(T)):
        alone = vits.decode(codes[b].view(1, 1, -1), text[b][None], refers[b], noise=noise[b].T[None])[0, 0]
        assert batch[b].shape == alone.shape == (2 * T[b] * 640,)
        assert rel(batch[b], alone) < TOL_WAVE, b
        assert rel(batch[b][-4096:], alone[-4096:]) < TOL_WAVE, b                       # no padding leaks into the tail
    # row 2 (the shortest) beside long rows and beside a short one
    among_long = vits.decode_batch([codes[2], codes[1], codes[3]], [text[2], text[1], text[3]], ge[[2, 1, 3]],
                                   noise=[noise[2], noise[1], noise[3]])[0]
    among_short = vits.decode_batch([codes[2], codes[2][:4]], [text[2], text[2][:3]], ge[[2, 0]],
                                    noise=[noise[2], noise[2][:8]])[0]
    assert rel(among_long, among_short) < TOL_WAVE and rel(among_long, batch[2]) < TOL_WAVE
