"""GPU tests of batched AR decoding (`pytest -m gpu`): the row Linear, the per-row-key decode attention and the fused sampler
against float64 / the torch oracle, row independence of the token step, and Text2SemanticDecoder.infer_panel_batch_infer end to
end against the tokens the reference decoded (tests/golden/infer_batch.json)."""
import json
import math
import os

import pytest
import torch

from oracle import gpt_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_batch.json")))
DEV = torch.device("cuda", 0)
TOL_NET = 3e-3
V, EOS, D = 1025, 1024, 512


@pytest.fixture(scope="module")
def ops():
    from easevoice_trainer_b200 import lib, ops
    lib.init().evk_set_precise(0)
    return ops


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _packed(ops, N, C, g):
    wv = (torch.randn(N, C, 1, generator=g) / math.sqrt(C)).to(DEV)
    return ops.pack_weight(wv, None, need_pb=False), torch.randn(N, generator=g).to(DEV)


@pytest.mark.parametrize("N,C", [(1536, 512), (512, 512), (2048, 512), (512, 2048), (1028, 512)])
def test_linear_rows_many_rows(ops, N, C):
    g = torch.Generator().manual_seed(N + C)
    pw, bias = _packed(ops, N, C, g)
    wr = pw.pa[0, :N, :C].double().cpu()
    xs = torch.randn(64, C, generator=g).to(DEV)
    with torch.no_grad():
        full = ops.linear_rows(xs.view(64, 1, C), pw, bias, act=ops.ACT_RELU)
        for rows in (5, 8, 16, 33, 64):
            y = ops.linear_rows(xs[:rows].view(rows, 1, C), pw, bias, act=ops.ACT_RELU)
            ref = torch.relu(xs[:rows].double().cpu() @ wr.t() + bias.double().cpu())
            assert rel(y.view(rows, N), ref) < 2e-6, rows
            assert torch.equal(y, full[:rows]), rows                # a row's result does not depend on the batch
        for rows in (1, 2, 3, 4):                                   # the <= 4-row launches (one staging chunk, as before)
            y = ops.linear(xs[:rows].view(1, rows, C), pw, bias, act=ops.ACT_RELU)
            assert torch.equal(y.view(rows, 1, N), full[:rows]), rows


def test_attention_with_per_row_key_ranges(ops):
    g = torch.Generator().manual_seed(5)
    B, max_len, H = 4, 40, 16
    xl = [40, 7, 23, 1]
    n_prev = 40 + 17 + 9                                            # text, prompt, 9 generated tokens before this one
    cache = torch.randn(B, 80, 3 * D, generator=g)
    for b in range(B):
        cache[b, xl[b]:max_len] = float("nan")                     # padding must never be read
    cache = cache.to(DEV)
    row = torch.randn(B, 1, 3 * D, generator=g).to(DEV)
    skip = torch.tensor([[v, max_len] for v in xl], dtype=torch.int32, device=DEV)
    n = torch.tensor([n_prev], dtype=torch.int32, device=DEV)
    out = ops.attn_decode_dev(cache, n, H, row, skip)
    c = cache.double().cpu()
    for b in range(B):
        keys = list(range(xl[b])) + list(range(max_len, n_prev + 1))
        q = c[b, n_prev, :D].view(H, 1, 32)
        k = c[b, keys, D:2 * D].view(-1, H, 32).transpose(0, 1)
        v = c[b, keys, 2 * D:].view(-1, H, 32).transpose(0, 1)
        ref = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32.0), -1) @ v).reshape(D)
        assert rel(out[b, 0], ref) < 2e-6, b


def _net(eos_scale=1.0, n_layer=None):
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    c = GOLD["cfg"]
    m = dict(gpt_oracle.GPT_MODEL, n_layer=n_layer or c["n_layer"])
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), c["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][m["EOS"]] *= eos_scale
    net = Text2SemanticDecoder({"model": m})
    net.load_state_dict(P)
    return net.to(DEV).eval()


def test_token_step_rows_are_independent(ops):
    net = _net()
    g = torch.Generator().manual_seed(9)
    B, rows, n_prev = 6, 64, 45
    caches = [torch.randn(B, rows, 3 * D, generator=g).to(DEV) for _ in range(net.num_layers)]
    x = torch.randn(B, 1, D, generator=g).to(DEV)
    skip = torch.tensor([[10, 20]] * B, dtype=torch.int32, device=DEV)

    def run(cs, xx):
        n = torch.tensor([n_prev], dtype=torch.int32, device=DEV)
        net._active, net._memo_pack = net.packed_for_inference(), True
        try:
            with torch.no_grad():
                h = xx
                for i in range(net.num_layers):
                    h = net._infer_layer(i, h, cs[i], n, skip=skip)
                return ops.linear_rows(h, net.w("ar_predict_layer", pad0=1028))
        finally:
            net._active, net._memo_pack = None, False
    a = run([c.clone() for c in caches], x)
    c2 = [c.clone() for c in caches]
    for c in c2:
        c[2] = torch.randn(rows, 3 * D, generator=g).to(DEV)
    x2 = x.clone()
    x2[2] = torch.randn(1, D, generator=g).to(DEV)
    b = run(c2, x2)
    keep = [0, 1, 3, 4, 5]
    assert torch.equal(a[keep], b[keep]) and not torch.equal(a[2], b[2])


class Sampler:
    """Device buffers of one evk_sample_tokens call on B rows."""

    def __init__(self, ops, logits, hists, prefix, step, top_k, top_p, T, pen, seed=0, q=None):
        B = logits.shape[0]
        self.ops, self.logits, self.q = ops, logits.to(DEV).contiguous(), None if q is None else q.to(DEV).contiguous()
        self.hist = torch.zeros(B, prefix + step + 4, dtype=torch.int64, device=DEV)
        seen = torch.zeros(B, 33 * 32, dtype=torch.int64)
        for b, h in enumerate(hists):
            if h:
                self.hist[b, :len(h)] = torch.tensor(h)
                seen[b, h] = 1
        words = (seen.view(B, 33, 32) << torch.arange(32)).sum(-1)
        self.seen = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32).to(DEV)
        self.fin = torch.full((B, 2), -1, dtype=torch.int32, device=DEV)
        n0 = 100
        self.n = torch.tensor([n0 + step], dtype=torch.int32, device=DEV)
        self.icfg = torch.tensor([seed, prefix, n0, top_k, -1, 1500], dtype=torch.int64, device=DEV)
        self.fcfg = torch.tensor([top_p, T, pen], dtype=torch.float32, device=DEV)
        gg = torch.Generator().manual_seed(1)
        self.emb = torch.randn(V, D, generator=gg).to(DEV)
        self.pe = torch.randn(prefix + step + 4, D, generator=gg).to(DEV)
        self.alpha = torch.tensor([1.3], device=DEV)
        self.x = torch.zeros(B, 1, D, device=DEV)
        self.prefix, self.step = prefix, step

    def __call__(self):
        self.ops.sample_tokens(self.logits, V, EOS, self.icfg, self.fcfg, self.n, self.hist, self.seen, self.fin, self.emb, self.pe,
                               self.alpha, self.x, q=self.q)
        torch.cuda.synchronize()
        return self.hist[:, self.prefix + self.step].cpu(), self.fin.cpu()


@pytest.mark.parametrize("step", [0, 3])
@pytest.mark.parametrize("pen", [1.0, 1.35])
@pytest.mark.parametrize("T", [0.8, 1.0, 1.3])
@pytest.mark.parametrize("top_p", [1.0, 0.9, 0.6])
@pytest.mark.parametrize("top_k", [1, 5, 15])
def test_sampler_with_supplied_draws_matches_oracle(ops, top_k, top_p, T, pen, step):
    g = torch.Generator().manual_seed(top_k * 1000 + int(top_p * 100) + int(T * 10) + int(pen * 100) + step)
    B, prefix = 12, 9
    logits = torch.randn(B, V, generator=g) * 2.5
    logits[:4, EOS] = logits[:4].max(-1).values + 1.0               # rows 0-3: EOS is the argmax (stops unless step 0)
    logits[4:6, :8] += 4.0                                          # rows 4-5: the history's tokens lead, the penalty matters
    hists = [torch.randint(0, 1024, (prefix + step,), generator=g).tolist() for _ in range(B)]
    for b in range(4, 8):
        hists[b][1:4] = [hists[b][0]] * 3                           # repeats
        hists[b][4:8] = list(range(4))
    q = torch.empty(B, V).exponential_(1, generator=g)
    s = Sampler(ops, logits, hists, prefix, step, top_k, top_p, T, pen, q=q)
    tok, fin = s()
    for b in range(B):
        lb = logits[b:b + 1].clone()
        if step == 0:
            lb = lb[:, :-1]
        probs = gpt_oracle.logits_to_probs(lb, torch.tensor([hists[b]]), temperature=T, top_k=top_k, top_p=top_p, repetition_penalty=pen)
        want = int(torch.argmax(probs / q[b:b + 1, :probs.shape[1]], -1))
        eos = want == EOS or int(torch.argmax(lb, -1)) == EOS
        assert int(tok[b]) == want, (b, int(tok[b]), want)
        assert fin[b].tolist() == ([step, step - 1] if eos else [-1, -1]), (b, fin[b].tolist(), eos)
        if not eos:
            ref_x = s.emb[want] + s.alpha * s.pe[prefix + step]
            assert torch.equal(s.x[b, 0], ref_x), b
    if step == 0:
        assert (fin[:, 0] == -1).all()                             # EOS is excluded at step 0
    else:
        assert (fin[:4, 0] == step).all()


def test_sampler_generator_seed_and_distribution(ops):
    g = torch.Generator().manual_seed(3)
    row = torch.randn(1, V, generator=g) * 1.5
    B = 4096
    logits = row.expand(B, -1)

    def draw(seed):
        return Sampler(ops, logits, [[]] * B, 0, 1, 15, 1.0, 1.0, 1.0, seed=seed)()[0]
    t1, t2, t3 = draw(11), draw(11), draw(12)
    assert torch.equal(t1, t2) and not torch.equal(t1, t3)
    p = gpt_oracle.logits_to_probs(row.clone(), None, temperature=1.0, top_k=15)[0].double()
    support = torch.nonzero(p > 0).flatten()
    assert set(t1.tolist()) <= set(support.tolist())
    from scipy.stats import chisquare
    for t in (t1, t3):
        obs = torch.bincount(t, minlength=V)[support].double()
        assert chisquare(obs.numpy(), (p[support] / p[support].sum() * B).numpy()).pvalue > 0.001


def _inputs(padded=False):
    c = GOLD["cfg"]
    g = torch.Generator().manual_seed(c["seed"])
    x = [torch.randint(0, 732, (n,), generator=g) for n in c["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in c["x_lens"]]
    prompts = torch.randint(0, 1024, (1, c["Yp"]), generator=g).expand(c["B"], -1)
    if padded:
        X = max(c["x_lens"])
        xt = torch.zeros(c["B"], X, dtype=torch.long)
        for b, n in enumerate(c["x_lens"]):
            xt[b, :n] = x[b]
        x, bert = xt, [torch.nn.functional.pad(t, (0, X - t.shape[1])) for t in bert]
        return x.to(DEV), [t.to(DEV) for t in bert], prompts.to(DEV)
    return [t.to(DEV) for t in x], [t.to(DEV) for t in bert], prompts.to(DEV)


def _greedy(net, max_len=None, padded=False, trace=None):
    c = GOLD["cfg"]
    x, bert, prompts = _inputs(padded)
    kw = {} if max_len is None else dict(max_len=max_len)
    if trace is not None:
        kw["trace"] = trace
    return net.infer_panel_batch_infer(x, torch.tensor(c["x_lens"]), prompts, bert, top_k=1, top_p=100,
                                       early_stop_num=c["early_stop_num"], temperature=1.0, repetition_penalty=c["repetition_penalty"], **kw)


def test_batch_infer_greedy_matches_reference(ops):
    c = GOLD["cfg"]
    net = _net(c["eos_scale"])
    tr = []
    y, idx = _greedy(net, trace=tr)
    assert all(t.dtype == torch.int64 and t.device.type == "cuda" and t.dim() == 1 for t in y) and all(isinstance(i, int) for i in idx)
    diverged = {}
    for b in range(c["B"]):
        toks, ref = y[b].cpu().tolist(), GOLD["tokens"][b]
        bad = next((i for i, (u, v) in enumerate(zip(toks, ref)) if u != v), None)
        if bad is None and len(toks) == len(ref):
            assert idx[b] == GOLD["idx"][b], b
            continue
        # exact fp32 token step, TF32 prompt pass: an argmax may flip only where the reference's own top-2 margin is noise-sized
        step = (bad if bad is not None else min(len(toks), len(ref))) - c["Yp"]
        assert GOLD["top2_margin"][b][step] < 2e-2, (b, step, GOLD["top2_margin"][b][step])
        diverged[b] = step
    for s, rows in GOLD["logits_step"].items():
        for b, ref in rows.items():
            b = int(b)
            if b not in diverged or int(s) <= diverged[b]:
                assert rel(tr[int(s)][b, GOLD["logit_ids"]], torch.tensor(ref)) < TOL_NET, (s, b)
    # results unchanged with more padding, and with a padded [B, X] tensor instead of lists
    for kw in (dict(max_len=c["max_len"] + 11), dict(padded=True)):
        y2, idx2 = _greedy(net, **kw)
        assert idx2 == idx and all(torch.equal(a, b) for a, b in zip(y, y2)), kw


def test_batch_of_one_matches_infer_panel_naive(ops):
    net = _net(1.0)                                                 # no EOS before early stop (tests/golden/infer_batch.json cfg)
    x, bert, prompts = _inputs()
    y, idx = net.infer_panel_batch_infer(x[:1], torch.tensor([x[0].shape[0]]), prompts[:1], bert[:1], top_k=1, early_stop_num=20)
    yn, idxn = net.infer_panel_naive(x[0].unsqueeze(0), torch.tensor([x[0].shape[0]]), prompts[:1], bert[0].unsqueeze(0), top_k=1,
                                     early_stop_num=20)
    assert torch.equal(y[0], yn[0]) and idx == [20] and idxn == 19    # at early stop the naive path returns idx - 1


def test_eos_window_of_infer_panel_with_a_prompt(ops):
    net = _net(1.0)
    with torch.no_grad():
        # the last LayerNorm's output then sums to D whatever its input, so EOS has the logit 0.1 * D = 51.2 at every step,
        # far above every other class
        net.P(f"h.layers.{net.num_layers - 1}.norm2.weight").fill_(1.0)
        net.P(f"h.layers.{net.num_layers - 1}.norm2.bias").fill_(1.0)
        net.P("ar_predict_layer.weight")[EOS].fill_(0.1)
    x, bert, prompts = _inputs()
    Yp = prompts.shape[1]
    y, idx = net.infer_panel(x[0].unsqueeze(0), torch.tensor([x[0].shape[0]]), prompts[:1], bert[0].unsqueeze(0), top_k=1,
                             early_stop_num=50)
    assert tuple(y.shape) == (1, Yp + 11) and idx == 10                # EOS excluded for the first 11 steps, taken at step 11
    yb, idxb = net.infer_panel_batch_infer(x[:1], torch.tensor([x[0].shape[0]]), prompts[:1], bert[:1], top_k=1, early_stop_num=50)
    assert yb[0].shape[0] == Yp + 1 and idxb == [0]                    # excluded at step 0 only: stops at step 1
    assert torch.equal(yb[0], y[0, :Yp + 1])


def test_sampled_infer_panel_repeats_under_manual_seed(ops):
    net = _net(1.0, n_layer=4)
    x, bert, prompts = _inputs()
    kw = dict(top_k=15, top_p=0.9, early_stop_num=40, temperature=1.0)
    runs = []
    for seed in (0, 0, 1):
        torch.manual_seed(seed)
        runs.append(net.infer_panel(x[0].unsqueeze(0), torch.tensor([x[0].shape[0]]), prompts[:1], bert[0].unsqueeze(0), **kw))
    (y0, i0), (y1, i1), (y2, _) = runs
    assert torch.equal(y0, y1) and i0 == i1
    assert not torch.equal(y0, y2)                                      # the noise does come from the seeded generator
    assert torch.equal(y0[0, :prompts.shape[1]], prompts[0]) and int(y0.max()) < EOS


def test_infer_panel_reuses_its_step_graph(ops):
    net = _net(1.0, n_layer=4)
    x, bert, prompts = _inputs()

    def one(n):                                                         # the first n phonemes of row 0
        return net.infer_panel(x[0][None, :n], torch.tensor([n]), prompts[:1], bert[0][None, :, :n], top_k=1, early_stop_num=20)
    n = x[0].shape[0]
    one(n)
    st = net.__dict__["_batch_st1"]
    graph = st["graphs"][11]
    one(n - 3)
    net.infer_panel_batch_infer(x, torch.tensor(GOLD["cfg"]["x_lens"]), prompts, bert, top_k=1, early_stop_num=20)   # B > 1
    one(n - 5)
    assert net.__dict__["_batch_st1"] is st and st["graphs"][11] is graph


def test_sampled_batch_of_16(ops):
    net = _net(1.0, n_layer=4)
    g = torch.Generator().manual_seed(4)
    B, Yp, E = 16, 13, 40
    xl = torch.randint(5, 30, (B,), generator=g)
    x = [torch.randint(0, 732, (int(n),), generator=g).to(DEV) for n in xl]
    bert = [torch.randn(1024, int(n), generator=g).to(DEV) for n in xl]
    prompts = torch.randint(0, 1024, (1, Yp), generator=g).expand(B, -1).to(DEV)
    torch.manual_seed(0)
    y, idx = net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=15, top_p=1, early_stop_num=E, temperature=1.0)
    torch.manual_seed(0)
    y2, idx2 = net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=15, top_p=1, early_stop_num=E, temperature=1.0)
    assert len(y) == B and idx == idx2 and all(torch.equal(a, b) for a, b in zip(y, y2))     # torch.manual_seed reproduces a run
    for b in range(B):
        assert torch.equal(y[b][:Yp], prompts[b]) and Yp <= y[b].shape[0] <= Yp + E
        assert int(y[b].min()) >= 0 and int(y[b].max()) < EOS
        gen = y[b].shape[0] - Yp
        assert idx[b] == gen - 1 or idx[b] == gen == E                # finished on EOS, or stopped at early_stop_num
