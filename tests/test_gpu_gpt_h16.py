"""GPU tests of the stage-1 GPT's 16-bit compute type (`pytest -m gpu`), for fp16 and bf16.

Kernel (evk_attn_decode_h16): the appended k and v bit for bit against torch's cast, the output within a per-element bound of
float64 on the rounded cache, skipped keys and rows past the position never read (NaN there), an item's bits independent of
the launch's other items.  Decoder: first and teacher-forced step logits against the float64 emulation (tests/gpt_h16_ref.py)
by rel-L2, greedy tokens against the emulation's penalised argmax, row invariance of the batched decoders, fp32 -> 16-bit ->
fp32 switching against fresh models, the cache's size and the peak memory.  TTS: run and run_many after
enable_half_precision, and enable_half_precision(False) restoring the fp32 results."""
import math

import numpy as np
import pytest
import torch

from oracle import gpt_oracle as O
from oracle import tts_oracle as to
from tests import gpt_h16_ref as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
EOS = 1024
DTYPES = [torch.float16, torch.bfloat16]
U32 = 2.0 ** -24
# rel-L2 of the logits (first and every teacher-forced step, worst step) against the float64 emulation under
# evk_set_precise(1): only the fp32 accumulation orders and the rare 16-bit roundings of activations that lie within an fp32
# ulp of a 16-bit midpoint differ.  Measured on an H100 80GB HBM3 (700 W), worst of the 4- and 24-layer configs, with and
# without a prompt: 8.6e-4 (fp16), 7.9e-3 (bf16); the largest logit error 3.5e-3 (fp16), 2.8e-2 (bf16).
TOL_LOGITS = {torch.float16: 2e-3, torch.bfloat16: 1.5e-2}
# evk_set_precise(0) (TF32 prompt-pass attention), 4 layers: measured 7.9e-4 (fp16), 4.4e-3 (bf16)
TOL_LOGITS_TF32 = {torch.float16: 5e-3, torch.bfloat16: 2e-2}
# top-2 margin of the emulation's penalised logits above which the greedy token must be its argmax: more than twice the
# largest logit error measured above, so a flip there is a defect, not rounding
TAU = {torch.float16: 0.01, torch.bfloat16: 0.08}


@pytest.fixture(scope="module")
def L():
    from easevoice_trainer_b200 import lib
    L = lib.init()
    before = L.evk_get_precise()
    L.evk_set_precise(1)
    yield L
    L.evk_set_precise(before)


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def bits(t):
    return t.view(torch.int16).cpu()


# ---- kernel -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_attn_decode_h16_kernel(L, dtype):
    from easevoice_trainer_b200 import ops
    g = torch.Generator().manual_seed(7)
    B, H, rows = 16, 16, 1300
    D = 32 * H
    for n_prev in (0, 1, 37, 130, 1100):
        skip = torch.zeros(B, 2, dtype=torch.int32)
        for b in range(B):
            if b % 3 and n_prev > 2:                        # every third item skips nothing, the others a random range
                s0 = int(torch.randint(0, n_prev - 1, (1,), generator=g))
                skip[b] = torch.tensor([s0, int(torch.randint(s0, n_prev, (1,), generator=g))])
        cache = torch.full((B, rows, 2 * D), float("nan")).to(dtype)
        cache[:, :n_prev] = torch.randn(B, n_prev, 2 * D, generator=g).to(dtype)
        for b in range(B):
            cache[b, skip[b, 0]:skip[b, 1]] = float("nan")      # never read
        row = torch.randn(B, 1, 3 * D, generator=g) * 1.5
        cache, row, skip_d = cache.to(DEV), row.to(DEV), skip.to(DEV)
        n = torch.tensor([n_prev], dtype=torch.int32, device=DEV)
        before = cache.clone()
        out = ops.attn_decode_h16(cache, n, H, row, skip_d)
        # the appended key: torch's cast of the row's k and v, and nothing else written
        assert torch.equal(bits(cache[:, n_prev]), bits(row[:, 0, D:].to(dtype))), n_prev
        others = torch.ones(rows, dtype=torch.bool)
        others[n_prev] = False
        assert torch.equal(bits(cache[:, others]), bits(before[:, others]))
        c = cache.double().cpu()
        r = row.double().cpu()[:, 0]
        for b in range(B):
            keys = [j for j in range(n_prev + 1) if not skip[b, 0] <= j < skip[b, 1]]
            q = (r[b, :D].float() * (1.0 / math.sqrt(32.0))).double().view(H, 1, 32)    # the kernel's fp32 q * scale
            k = c[b, keys, :D].view(-1, H, 32).transpose(0, 1)
            v = c[b, keys, D:].view(-1, H, 32).transpose(0, 1)
            ref = (torch.softmax(q @ k.transpose(-1, -2), -1) @ v).reshape(D)
            # per element: the fp32 score (32 FMAs) and the exp perturb each probability by at most gamma_36 S relatively,
            # S = max over keys of sum_i |q_i k_i|; the per-thread and merge sums add gamma_(n/128 + 40); twice both, times
            # max |v|, bounds the output's error
            S = float((q.abs() @ k.abs().transpose(-1, -2)).max())
            gam = lambda m: m * U32 / (1 - m * U32)                 # noqa: E731
            vmax = v.abs().amax(1).reshape(D)
            bound = 2 * (gam(36) * S + gam(len(keys) / 128 + 40)) * vmax
            err = (out[b, 0].double().cpu() - ref).abs()
            assert torch.all(err <= bound), (n_prev, b, float((err / bound).max()))
            # item b alone gives the bits it gives among 16
            alone = ops.attn_decode_h16(before[b:b + 1].clone(), n, H, row[b:b + 1], skip_d[b:b + 1])
            assert torch.equal(alone, out[b:b + 1]), (n_prev, b)


# ---- decoder ------------------------------------------------------------------------------------------------------------
def _params(n_layer, seed):
    m = dict(O.GPT_MODEL, n_layer=n_layer)
    P = O.init_params(O.gpt_param_spec(m), seed)
    P["ar_text_position.alpha"].fill_(0.8)
    P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][EOS] = 0.0                     # EOS logit 0: never the argmax, decoding runs to early stop
    return m, P


def _net(m, P, dtype):
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    net = Text2SemanticDecoder({"model": m})
    net.load_state_dict(P)
    return net.set_compute_type(dtype).to(DEV).eval()


def _row(seed, X, Yp):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 732, (X,), generator=g)
    bert = torch.randn(1024, X, generator=g)
    prompt = torch.randint(0, 1024, (Yp,), generator=g) if Yp else None
    return x, bert, prompt


def _decode_and_compare(net, m, P, dtype, prompt_free, steps):
    """infer_panel_naive greedy on one row, teacher-forced emulation on its tokens -> (worst rel-L2 over the trace, max
    |logit error|, number of tokens checked against the emulation's argmax)."""
    x, bert, prompt = _row(11, 37, 0 if prompt_free else 23)
    tr = []
    y, _ = net.infer_panel_naive(x[None].to(DEV), torch.tensor([37]), None if prompt is None else prompt[None].to(DEV),
                                 bert[None].to(DEV), top_k=1, early_stop_num=steps, trace=tr)
    Yp = 0 if prompt is None else prompt.shape[0]
    toks = y[0, Yp:].cpu().tolist()
    assert len(tr) == len(toks) + 1 and len(toks) >= steps - 1
    emu = R.teacher_forced(P, m, dtype, x, bert, prompt, toks)
    got = torch.cat(tr).double().cpu()
    worst = max(rel(got[s], emu[s]) for s in range(len(tr)))
    abs_err = float((got - emu).abs().max())
    hist = [] if prompt is None else prompt.tolist()
    checked = 0
    for s, t in enumerate(toks):
        lp = R.penalised(emu[s], hist, 1.35)
        if s < 11:
            lp = lp[:EOS]                                       # EOS excluded for the first 11 steps
        top2 = lp.topk(2).values
        if float(top2[0] - top2[1]) > TAU[dtype]:
            assert t == int(lp.argmax()), (s, t, int(lp.argmax()))
            checked += 1
        hist.append(t)
    return worst, abs_err, checked


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_layer", [4, 24])
def test_decoder_logits_and_greedy_tokens_against_emulation(L, dtype, n_layer):
    m, P = _params(n_layer, 5 + n_layer)
    net = _net(m, P, dtype)
    for prompt_free in (False, True):
        worst, abs_err, checked = _decode_and_compare(net, m, P, dtype, prompt_free, 24)
        print(f"\n[gpt_h16] {dtype} layers={n_layer} prompt_free={prompt_free}: worst step rel-L2 {worst:.3e}, max |err| "
              f"{abs_err:.3e}, {checked} greedy tokens checked")
        assert worst < TOL_LOGITS[dtype] and checked >= 1
    # the 16-bit cache is part of the state: [B, rows, 2 D] in the compute type
    st = net.__dict__["_batch_st1"]
    assert all(c.dtype == dtype and c.shape[2] == 2 * m["hidden_dim"] for c in st["caches"])


@pytest.mark.parametrize("dtype", DTYPES)
def test_decoder_against_emulation_in_tf32_mode(L, dtype):
    m, P = _params(4, 9)
    L.evk_set_precise(0)
    try:
        worst, abs_err, _ = _decode_and_compare(_net(m, P, dtype), m, P, dtype, False, 24)
    finally:
        L.evk_set_precise(1)
    print(f"\n[gpt_h16] {dtype} evk_set_precise(0): worst step rel-L2 {worst:.3e}, max |err| {abs_err:.3e}")
    assert worst < TOL_LOGITS_TF32[dtype]


def _batch(seed, B, Yp):
    g = torch.Generator().manual_seed(seed)
    xl = torch.randint(5, 40, (B,), generator=g)
    x = [torch.randint(0, 732, (int(n),), generator=g).to(DEV) for n in xl]
    bert = [torch.randn(1024, int(n), generator=g).to(DEV) for n in xl]
    prompts = torch.randint(0, 1024, (1, Yp), generator=g).expand(B, -1).to(DEV)
    return x, xl, bert, prompts


@pytest.mark.parametrize("dtype", DTYPES)
def test_row_alone_and_in_a_batch_of_16(L, dtype):
    m, P = _params(4, 3)
    net = _net(m, P, dtype)
    x, xl, bert, prompts = _batch(2, 16, 17)
    max_len = int(xl.max())
    tr = []
    y, idx = net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=1, early_stop_num=30, max_len=max_len, trace=tr)
    for b in (0, 5, 15):
        alone = []
        y1, idx1 = net.infer_panel_batch_infer(x[b:b + 1], xl[b:b + 1], prompts[b:b + 1], bert[b:b + 1], top_k=1, early_stop_num=30,
                                               max_len=max_len, trace=alone)
        assert torch.equal(y1[0], y[b]) and idx1[0] == idx[b]
        assert len(alone) <= len(tr) and all(torch.equal(alone[s][0], tr[s][b]) for s in range(len(alone))), b
    # prompt-free rows as well
    tr = []
    y, _ = net.infer_panel_naive_batched(x, xl, None, bert, top_k=1, early_stop_num=20, max_len=max_len, trace=tr)
    alone = []
    y1, _ = net.infer_panel_naive_batched(x[3:4], xl[3:4], None, bert[3:4], top_k=1, early_stop_num=20, max_len=max_len, trace=alone)
    assert torch.equal(y1[0], y[3]) and all(torch.equal(alone[s][0], tr[s][3]) for s in range(len(alone)))


def _groups(seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, (n, yp, top_k) in enumerate(((2, 31, 1), (3, 12, 15), (1, 0, 5))):
        lens = torch.randint(6, 30, (n,), generator=g).tolist()
        out.append(dict(rows=[torch.randint(0, 732, (v,), generator=g).to(DEV) for v in lens], lens=lens,
                        bert=[torch.randn(1024, v, generator=g).to(DEV) for v in lens], max_len=max(lens) + k,
                        prompt=torch.randint(0, 1024, (yp,), generator=g).to(DEV) if yp else None,
                        seed=torch.tensor([100 + k], device=DEV), eos_steps=1 if yp else 11, top_k=top_k, top_p=0.9,
                        temperature=1.0, repetition_penalty=1.35, early_stop_num=25 + 5 * k))
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_groups_alone_and_packed(L, dtype):
    m, P = _params(4, 4)
    net = _net(m, P, dtype)
    groups = _groups(6)
    tr = []
    ys, fin = net.decode_groups(groups, trace=tr)
    r0 = 0
    for gr in groups:
        alone = []
        ya, fa = net.decode_groups([gr], trace=alone)
        for j in range(len(gr["rows"])):
            b = r0 + j
            assert torch.equal(ya[j], ys[b]) and fa[j] == fin[b], b
            assert all(torch.equal(alone[s][j], tr[s][b]) for s in range(fin[b][0] + 1)), b
        r0 += len(gr["rows"])


def _greedy_batch(net, trace):
    x, xl, bert, prompts = _batch(8, 3, 11)
    return net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=1, early_stop_num=20, trace=trace)


def test_switching_compute_type_matches_fresh_models(L):
    m, P = _params(4, 12)
    net = _net(m, P, None)
    runs = []
    for dt in (None, torch.float16, None):
        tr = []
        y, _ = _greedy_batch(net.set_compute_type(dt), tr)
        runs.append((y, tr))
        assert all(c.dtype == (dt or torch.float32) for c in net.__dict__["_batch_st"]["caches"])
    fresh = {}
    for dt in (None, torch.float16):
        tr = []
        fresh[dt] = (_greedy_batch(_net(m, P, dt), tr)[0], tr)
    for (y, tr), dt in zip(runs, (None, torch.float16, None)):
        fy, ftr = fresh[dt]
        assert all(torch.equal(a, b) for a, b in zip(y, fy)) and len(tr) == len(ftr)
        assert all(torch.equal(a, b) for a, b in zip(tr, ftr)), dt
    assert not all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))    # the 16-bit run does differ


@pytest.mark.parametrize("dtype", DTYPES)
def test_peak_memory_drops_by_the_cache_difference(L, dtype):
    m, P = _params(24, 1)
    x, xl, bert, prompts = _batch(9, 16, 150)
    peaks = {}
    for dt in (None, dtype):
        net = _net(m, P, dt)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=1, early_stop_num=200)
        torch.cuda.synchronize()
        peaks[dt] = torch.cuda.max_memory_allocated() - base
        caches = net.__dict__["_batch_st"]["caches"]
        rows = caches[0].shape[1]
        assert all(c.dtype == (dt or torch.float32) and c.shape == (16, rows, (3 if dt is None else 2) * 512) for c in caches)
        del net, caches
        torch.cuda.empty_cache()
    diff = 24 * 16 * rows * (3 * 512 * 4 - 2 * 512 * 2)
    print(f"\n[gpt_h16] {dtype} B=16 peak {peaks[None] / 2**30:.3f} GiB (fp32) -> {peaks[dtype] / 2**30:.3f} GiB, "
          f"cache difference {diff / 2**30:.3f} GiB")
    assert peaks[None] - peaks[dtype] >= diff


# ---- TTS ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tts_mod(L):
    from easevoice_trainer_b200 import tts
    return tts


def test_tts_run_and_run_many_in_half_precision(tts_mod, files):
    from tests.test_gpu_tts import _models
    from tests.test_gpu_tts_many import REQS, _Caller, _inputs
    tts = tts_mod
    paths, clips = files
    obj = _Caller(tts, _models(), paths, clips)
    reqs = [_inputs(paths, i) for i in range(len(REQS))]

    def runs():
        out, codes = [], []
        for r in reqs:
            obj.codes.clear()
            out.append(list(tts.run(obj, r)))
            codes.append(list(obj.codes))
        return out, codes
    fp32, codes32 = runs()
    tts.enable_half_precision(obj, save=False)
    assert obj.configs.is_half and obj.precision is torch.float16 and obj.t2s_model.model.compute_type is torch.float16
    half, codes16 = runs()
    for outs in half:
        assert outs and all(sr == to.SR and a.dtype == np.int16 and a.size > 0 for sr, a in outs)
    st = [v for k, v in obj.t2s_model.model.__dict__.items() if k in ("_batch_st", "_batch_st1")]
    assert st and all(c.dtype == torch.float16 for s in st for c in s["caches"])     # the AR decoder did run in 16 bits
    obj.codes.clear()
    results, errors = tts.run_many(obj, reqs)
    assert errors == [] and len(results) == len(reqs)
    assert sorted(obj.codes) == sorted(sum(codes16, []))          # each request's tokens are those of its own run
    tts.enable_half_precision(obj, False, save=False)
    assert obj.t2s_model.model.compute_type is None
    back, codes_back = runs()
    assert codes_back == codes32
    for a, b in zip(back, fp32):
        assert len(a) == len(b) and all(sa == sb and np.array_equal(xa, xb) for (sa, xa), (sb, xb) in zip(a, b))


@pytest.fixture()
def files():
    import os
    import tempfile
    from tests.test_gpu_tts_many import _clip
    with tempfile.TemporaryDirectory() as d:
        clips = {f"c{i}.wav": _clip(40 + i, s) for i, s in enumerate((3.2, 4.5, 6.1, 8.0, 3.6))}
        paths = {}
        for n in clips:
            paths[n] = os.path.join(d, n)
            open(paths[n], "wb").close()
        yield paths, clips
