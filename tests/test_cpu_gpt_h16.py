"""CPU tests of the stage-1 GPT's 16-bit compute type: set_compute_type's validation and the packed-weight cache key following
it, tts.enable_half_precision on a stand-in TTS object, the float64 decoding emulation (tests/gpt_h16_ref.py) against a direct
whole-sequence computation and against the fp32 oracle, and round-to-nearest-even at exact fp16 and bf16 midpoints of the
torch cast that fills the 16-bit K/V cache in the prompt pass."""
import types

import numpy as np
import pytest
import torch

from oracle import gpt_oracle as O
from tests import gpt_h16_ref as R

TINY = dict(O.GPT_MODEL, hidden_dim=64, embedding_dim=64, head=2, linear_units=256, n_layer=2)


def _net():
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    return Text2SemanticDecoder({"model": TINY})


def test_set_compute_type_validation_and_cache_key():
    net = _net()
    sd0 = {k: v.clone() for k, v in net.state_dict().items()}
    k0 = net.weights_key()
    built = []
    net.cached("probe", lambda: built.append(1))
    net.cached("probe", lambda: built.append(1))
    assert len(built) == 1 and net.compute_type is None
    for dt in (torch.float16, torch.bfloat16):
        assert net.set_compute_type(dt) is net and net.compute_type is dt
        assert net.weights_key() != k0
        net.cached("probe", lambda: built.append(1))
    assert len(built) == 3
    assert net.set_compute_type(None) is net and net.weights_key() == k0
    for bad in (torch.float32, "float16", torch.int8, 16):
        with pytest.raises(ValueError):
            net.set_compute_type(bad)
    assert net.compute_type is None
    net.set_compute_type(torch.float16)
    sd = net.state_dict()                                   # parameters stay fp32: the state dict does not change
    assert sd.keys() == sd0.keys() and all(sd[k].dtype == torch.float32 and torch.equal(sd[k], sd0[k]) for k in sd)


def _tts(device):
    saved = []
    others = dict(vits_model=object(), bert_model=object(), cnhuhbert_model=object())
    t = types.SimpleNamespace(configs=types.SimpleNamespace(device=device, is_half=False, save_configs=lambda: saved.append(1)),
                              precision=torch.float32, t2s_model=types.SimpleNamespace(model=_net()), **others)
    return t, saved, others


def test_enable_half_precision():
    from easevoice_trainer_b200 import tts
    t, saved, others = _tts("cpu")
    tts.enable_half_precision(t)                            # on a CPU device enabling changes nothing
    assert t.configs.is_half is False and t.precision is torch.float32 and saved == [] and t.t2s_model.model.compute_type is None
    for dev in ("cuda", torch.device("cuda", 0)):
        t, saved, others = _tts(dev)
        tts.enable_half_precision(t)
        assert t.configs.is_half is True and t.precision is torch.float16 and saved == [1]
        assert t.t2s_model.model.compute_type is torch.float16
        tts.enable_half_precision(t, False, save=False)
        assert t.configs.is_half is False and t.precision is torch.float32 and saved == [1]
        assert t.t2s_model.model.compute_type is None
        tts.enable_half_precision(t, True, save=False)
        assert t.t2s_model.model.compute_type is torch.float16 and saved == [1]
        assert all(getattr(t, k) is v for k, v in others.items())      # the vocoder, BERT and HuBERT are left alone


def _direct(P, m, dtype, x, bert, prompt, tokens):
    """The decoder's logits computed over the whole sequence at once, layer by layer: prompt positions attend the unrounded
    k / v under the prefix-LM mask, generated positions the rounded k / v of every position up to their own."""
    P = R.rounded(P, dtype)
    D, H = m["hidden_dim"], m["head"]
    X, Yp, S = x.shape[0], 0 if prompt is None else prompt.shape[0], len(tokens)
    L0 = X + Yp
    pe = O.sine_pe(L0 + S + 8, D).double()
    y = torch.cat([torch.zeros(0, dtype=torch.long) if prompt is None else prompt, torch.tensor(tokens, dtype=torch.long)])
    h = torch.cat([P["ar_text_embedding.word_embeddings.weight"][x] + R.lin(bert.T, P["bert_proj.weight"], P["bert_proj.bias"], dtype)
                   + P["ar_text_position.alpha"] * pe[:X],
                   P["ar_audio_embedding.word_embeddings.weight"][y] + P["ar_audio_position.alpha"] * pe[:Yp + S]])
    mask = O.prefix_lm_mask(torch.tensor([X]), torch.tensor([Yp]), X, Yp)[0]
    for i in range(m["n_layer"]):
        p = f"h.layers.{i}."
        q, k, v = R.lin(h, P[p + "self_attn.in_proj_weight"], P[p + "self_attn.in_proj_bias"], dtype).split(D, -1)
        kr, vr = R.h16(k, dtype), R.h16(v, dtype)
        a = torch.cat([R._attend(q[:L0], k[:L0], v[:L0], H, mask)]
                      + [R._attend(q[t:t + 1], kr[:t + 1], vr[:t + 1], H) for t in range(L0, L0 + S)])
        h = R._ffn(P, p, h, a, dtype)
    return R.lin(h[L0 - 1:], P["ar_predict_layer.weight"], None, dtype)


def _inputs(seed, X, Yp):
    g = torch.Generator().manual_seed(seed)
    P = O.init_params(O.gpt_param_spec(TINY), seed)
    x = torch.randint(0, 732, (X,), generator=g)
    bert = torch.randn(1024, X, generator=g)
    prompt = torch.randint(0, 1024, (Yp,), generator=g) if Yp else None
    tokens = torch.randint(0, 1024, (6,), generator=g).tolist()
    return P, x, bert, prompt, tokens


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, None])
@pytest.mark.parametrize("Yp", [0, 5])
def test_emulation_against_direct_float64(dtype, Yp):
    P, x, bert, prompt, tokens = _inputs(3 + Yp, 9, Yp)
    got = R.teacher_forced(P, TINY, dtype, x, bert, prompt, tokens)
    want = _direct(P, TINY, dtype, x, bert, prompt, tokens)
    assert got.shape == (7, TINY["vocab_size"])
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    if dtype is not None:                                   # the rounding is real: not the unrounded computation
        assert float((got - R.teacher_forced(P, TINY, None, x, bert, prompt, tokens)).abs().max()) > 1e-4


def test_unrounded_emulation_matches_fp32_oracle():
    """dtype None against gpt_oracle.infer_panel, which recomputes the whole sequence every step (greedy, so its tokens are
    deterministic): the prompt pass, the step positions and the first-logits row agree."""
    P, x, bert, prompt, _ = _inputs(4, 9, 5)
    trace = []
    y, _ = O.infer_panel(P, x[None], bert[None], prompt[None], top_k=1, m=TINY, max_steps=6, trace=trace)
    tokens = y[0, prompt.shape[0]:].tolist()
    assert len(trace) == len(tokens) + 1
    got = R.teacher_forced(P, TINY, None, x, bert, prompt, tokens)
    ref = torch.cat(trace).double()
    assert float((got - ref).norm() / ref.norm()) < 1e-5


def rne_bf16(a):
    """fp32 -> bf16 by round to nearest even on the bit pattern, as float64."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


@pytest.mark.parametrize("dtype,ulp", [(torch.float16, 2.0 ** -10), (torch.bfloat16, 2.0 ** -7)])
def test_cache_cast_rounds_to_nearest_even_at_midpoints(dtype, ulp):
    """The prompt pass fills the 16-bit cache with torch's copy_ cast.  1 + ulp/2 lies halfway between 1 (even) and 1 + ulp:
    RNE gives 1.  1 + 3 ulp/2 lies between 1 + ulp (odd) and 1 + 2 ulp (even): RNE gives 1 + 2 ulp, truncation 1 + ulp."""
    x = torch.tensor([1 + ulp / 2, 1 + 3 * ulp / 2, -(1 + 3 * ulp / 2), 1 + 3 * ulp / 2 + ulp / 64, 3 * 2.0 ** -20], dtype=torch.float32)
    manual = x.numpy().astype(np.float16).astype(np.float64) if dtype is torch.float16 else rne_bf16(x.numpy())
    assert np.array_equal(manual[:4], [1.0, 1 + 2 * ulp, -(1 + 2 * ulp), 1 + 2 * ulp])
    cache = torch.empty(2, 5, dtype=dtype)
    cache.copy_(x[None].expand(2, -1))
    assert np.array_equal(cache.double().numpy(), np.stack([manual, manual]))
    assert torch.equal(R.h16(x, dtype), torch.from_numpy(manual))
