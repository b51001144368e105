"""GPU tests of prompt-free AR decoding (`pytest -m gpu`): the text-only prompt pass kernels (empty audio part), the sampler's EOS
window (evk_sample_tokens), Text2SemanticDecoder.infer_panel_naive(prompts=None) and the batched
infer_panel_naive_batched(prompts=None) against the tokens the reference decoded (tests/golden/infer_ref_free.json) and
against each other."""
import json
import math
import os

import pytest
import torch

from oracle import gpt_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_ref_free.json")))
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


def test_text_only_prompt_pass_kernels(ops):
    g = torch.Generator().manual_seed(21)
    B, L, H = 3, 70, 16                                              # 70: the second key / query tile is partial
    xl = [70, 33, 1]
    qkv = torch.randn(B, L, 3 * D, generator=g).to(DEV)
    xlen = torch.tensor(xl, device=DEV)
    out = ops.flash_attention(qkv, heads=H, prefix=L, xlen=xlen, ylen=torch.zeros(B, dtype=torch.int64, device=DEV))
    c = qkv.double().cpu()
    for b in range(B):                                               # every query sees its row's text, nothing else
        q, k, v = [c[b, :, i * D:(i + 1) * D].view(L, H, 32).transpose(0, 1) for i in range(3)]
        s = q @ k[:, :xl[b]].transpose(-1, -2) / math.sqrt(32.0)
        ref = (torch.softmax(s, -1) @ v[:, :xl[b]]).transpose(0, 1).reshape(L, D)
        assert rel(out[b], ref) < 5e-3, b                            # TF32 products
    # an empty audio part through the embedding and the positional concat
    table = torch.randn(V, D, generator=g).to(DEV)
    ye = ops.embedding(table, torch.zeros((B, 0), dtype=torch.int64, device=DEV))
    assert tuple(ye.shape) == (B, 0, D)
    xe = torch.randn(B, 9, D, generator=g).to(DEV)
    pe = torch.randn(16, D, generator=g).to(DEV)
    ax, ay = torch.tensor([0.8], device=DEV), torch.tensor([1.3], device=DEV)
    h = ops.gpt_embed(xe, ye, ax, ay, pe)
    assert tuple(h.shape) == (B, 9, D) and rel(h, xe + 0.8 * pe[:9]) < 1e-6


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


def _inputs():
    c = GOLD["cfg"]
    g = torch.Generator().manual_seed(c["seed"])
    x = [torch.randint(0, 732, (n,), generator=g) for n in c["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in c["x_lens"]]
    return [t.to(DEV) for t in x], [t.to(DEV) for t in bert]


def _check_against_golden(y, traces):
    """y[b]: 1-D tokens of row b; traces[b][s]: the [V] logits of row b at step s.  Tokens identical, except that an argmax may
    flip where the reference's own top-2 margin is noise-sized (exact fp32 token step, TF32 prompt pass); logits within TOL_NET
    up to the first divergence."""
    c = GOLD["cfg"]
    diverged = {}
    for b in range(c["B"]):
        toks, ref = y[b].cpu().tolist(), GOLD["tokens"][b]
        bad = next((i for i, (u, v) in enumerate(zip(toks, ref)) if u != v), None)
        if bad is None and len(toks) == len(ref):
            continue
        step = bad if bad is not None else min(len(toks), len(ref))
        assert GOLD["top2_margin"][b][step] < 2e-2, (b, step, GOLD["top2_margin"][b][step])
        diverged[b] = step
    for s, rows in GOLD["logits_step"].items():
        for b, ref in rows.items():
            b = int(b)
            if b not in diverged or int(s) <= diverged[b]:
                assert rel(traces[b][int(s)][GOLD["logit_ids"]], torch.tensor(ref)) < TOL_NET, (s, b)
    return diverged


def _per_row(net, x, bert, **kw):
    c = GOLD["cfg"]
    ys, traces = [], []
    for b in range(len(x)):
        tr = []
        y, idx = net.infer_panel_naive(x[b].unsqueeze(0), torch.tensor([x[b].shape[0]]), None, bert[b].unsqueeze(0), top_k=1,
                                       early_stop_num=c["early_stop_num"], trace=tr, **kw)
        assert idx == 0 and y.dim() == 2 and y.shape[0] == 1 and y.dtype == torch.int64 and y.device.type == "cuda"
        ys.append(y[0])
        traces.append([t[0] for t in tr])
    return ys, traces


def _batched(net, x, bert, max_len=None, trace=None, **kw):
    c = GOLD["cfg"]
    kw = dict(kw)
    if max_len is not None:
        kw["max_len"] = max_len
    if trace is not None:
        kw["trace"] = trace
    return net.infer_panel_naive_batched(x, torch.tensor([t.shape[0] for t in x]), None, bert, top_k=1, early_stop_num=c["early_stop_num"],
                                         **kw)


def test_single_utterance_matches_reference(ops):
    net = _net(GOLD["cfg"]["eos_scale"])
    x, bert = _inputs()
    y, traces = _per_row(net, x, bert)
    _check_against_golden(y, traces)


def test_batched_matches_reference_and_per_row_path(ops):
    c = GOLD["cfg"]
    net = _net(c["eos_scale"])
    x, bert = _inputs()
    tr = []
    y, idx = _batched(net, x, bert, trace=tr)
    assert idx == [0] * c["B"]
    assert all(t.dtype == torch.int64 and t.device.type == "cuda" and t.dim() == 1 for t in y)
    _check_against_golden(y, [[t[b] for t in tr] for b in range(c["B"])])
    y1, _ = _per_row(net, x, bert)
    assert all(torch.equal(a, b) for a, b in zip(y, y1))
    # TTS-shaped call (unpadded rows, max_len in kwargs) with a wider max_len: same results
    y2, idx2 = _batched(net, x, bert, max_len=max(c["x_lens"]) + 11)
    assert idx2 == idx and all(torch.equal(a, b) for a, b in zip(y, y2))


def test_batch_infer_forwards_at_the_default_penalty(ops):
    c = GOLD["cfg"]
    net = _net(c["eos_scale"])
    x, bert = _inputs()
    xl = torch.tensor(c["x_lens"])
    # t2s_model.py:576-578: repetition_penalty is not passed on, so 1.35 applies whatever the caller gives
    y, idx = net.infer_panel_batch_infer(x, xl, None, bert, top_k=1, early_stop_num=c["early_stop_num"], repetition_penalty=2.0)
    y2, idx2 = net.infer_panel_naive_batched(x, xl, None, bert, top_k=1, early_stop_num=c["early_stop_num"])
    assert idx == idx2 == [0] * c["B"] and all(torch.equal(a, b) for a, b in zip(y, y2))
    # a decode with a prompt on the same batch state (its own step graph, EOS window 1) leaves the prompt-free results unchanged
    prompts = torch.randint(0, 1024, (1, 7), generator=torch.Generator().manual_seed(2)).expand(c["B"], -1).to(DEV)
    net.infer_panel_batch_infer(x, xl, prompts, bert, top_k=1, early_stop_num=c["early_stop_num"])
    y3, _ = net.infer_panel_naive_batched(x, xl, None, bert, top_k=1, early_stop_num=c["early_stop_num"])
    assert all(torch.equal(a, b) for a, b in zip(y, y3))


class _Sampler:
    """Device buffers of one sampler call on B rows at step `step` (prefix 0, as in prompt-free decoding)."""

    def __init__(self, ops, logits, step, q):
        B = logits.shape[0]
        self.ops, self.logits, self.q = ops, logits.to(DEV).contiguous(), q.to(DEV).contiguous()
        self.hist = torch.zeros(B, step + 4, dtype=torch.int64, device=DEV)
        self.seen = torch.zeros(B, 33, dtype=torch.int32, device=DEV)
        self.fin = torch.full((B, 2), -1, dtype=torch.int32, device=DEV)
        self.n = torch.tensor([100 + step], dtype=torch.int32, device=DEV)
        self.icfg = torch.tensor([0, 0, 100, 15, -1, 1500], dtype=torch.int64, device=DEV)
        self.fcfg = torch.tensor([1.0, 1.0, 1.35], dtype=torch.float32, device=DEV)
        gg = torch.Generator().manual_seed(1)
        self.emb = torch.randn(V, D, generator=gg).to(DEV)
        self.pe = torch.randn(step + 4, D, generator=gg).to(DEV)
        self.alpha = torch.tensor([1.3], device=DEV)
        self.x = torch.zeros(B, 1, D, device=DEV)
        self.step = step

    def ex(self, eos_steps):
        self.ops.sample_tokens(self.logits, V, EOS, self.icfg, self.fcfg, self.n, self.hist, self.seen, self.fin, self.emb, self.pe,
                               self.alpha, self.x, q=self.q, eos_steps=eos_steps)
        return self.result()

    def plain(self):                                                 # the entry point called directly with eos_steps = 1
        p = self.ops._p
        self.ops._call("evk_sample_tokens", p(self.logits), self.logits.stride(0), self.logits.shape[0], V, EOS, 1, p(self.icfg),
                       p(self.fcfg), p(self.n), p(self.q), self.q.stride(0), p(self.hist), self.hist.stride(0), p(self.seen),
                       p(self.fin), p(self.emb), p(self.pe), p(self.alpha), p(self.x), D)
        return self.result()

    def result(self):
        torch.cuda.synchronize()
        return self.hist[:, self.step].cpu(), self.fin.cpu(), self.x.cpu()


def test_sampler_eos_steps_window(ops):
    g = torch.Generator().manual_seed(8)
    B = 8
    logits = torch.randn(B, V, generator=g) * 2.5
    logits[:4, EOS] = logits[:4].max(-1).values + 1.0               # rows 0-3: EOS is the argmax
    logits[4:, EOS] = logits[4:].min(-1).values - 1.0               # rows 4-7: EOS cannot be sampled
    q = torch.empty(B, V).exponential_(1, generator=g)
    tok, fin, _ = _Sampler(ops, logits, 10, q).ex(11)                # step 10 lies inside an 11-step window: nobody stops
    assert (fin == -1).all() and (tok < EOS).all()
    _, fin, _ = _Sampler(ops, logits, 11, q).ex(11)                  # step 11: the EOS rows stop, (idx, idx - 1)
    assert fin[:4].tolist() == [[11, 10]] * 4 and (fin[4:] == -1).all()
    _, fin, _ = _Sampler(ops, logits, 10, q).ex(1)                   # a 1-step window stops them at step 10 already
    assert fin[:4].tolist() == [[10, 9]] * 4
    for step in (0, 3):                                              # eos_steps = 1 is the batched decoders' call
        a, b = _Sampler(ops, logits, step, q).ex(1), _Sampler(ops, logits, step, q).plain()
        assert all(torch.equal(u, v) for u, v in zip(a, b)), step
    with pytest.raises(ValueError, match="eos_steps"):
        _Sampler(ops, logits, 0, q).ex(-1)


def _random_rows(B, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    xl = torch.randint(lo, hi, (B,), generator=g)
    x = [torch.randint(0, 732, (int(n),), generator=g).to(DEV) for n in xl]
    bert = [torch.randn(1024, int(n), generator=g).to(DEV) for n in xl]
    return x, xl, bert


def test_sampled_batch_of_16(ops):
    net = _net(1.3, n_layer=4)
    B, E = 16, 40
    x, xl, bert = _random_rows(B, 5, 30, 4)
    torch.manual_seed(0)
    y, idx = net.infer_panel_naive_batched(x, xl, None, bert, top_k=15, top_p=1, early_stop_num=E, temperature=1.0)
    torch.manual_seed(0)
    y2, idx2 = net.infer_panel_naive_batched(x, xl, None, bert, top_k=15, top_p=1, early_stop_num=E, temperature=1.0)
    assert len(y) == B and idx == idx2 == [0] * B and all(torch.equal(a, b) for a, b in zip(y, y2))  # manual_seed reproduces a run
    for b in range(B):
        n = y[b].shape[0]
        # stopped at early_stop_num (E tokens), or on EOS, which the first 11 steps exclude (11 <= n < E)
        assert 11 <= n <= E, (b, n)
        assert int(y[b].min()) >= 0 and int(y[b].max()) < EOS


def test_batch_of_70_runs_in_chunks(ops):
    net = _net(1.0)
    B, E = 70, 12
    x, xl, bert = _random_rows(B, 3, 20, 6)
    y, idx = net.infer_panel_naive_batched(x, xl, None, bert, top_k=1, early_stop_num=E)
    assert len(y) == B and idx == [0] * B and all(t.shape[0] <= E for t in y)
    y2, _ = net.infer_panel_naive_batched(x[64:], xl[64:], None, bert[64:], top_k=1, early_stop_num=E)
    assert all(torch.equal(a, b) for a, b in zip(y[64:], y2))


def test_early_stop_zero_returns_empty_rows(ops):
    net = _net(1.0)
    x, bert = _inputs()
    y, idx = net.infer_panel_naive(x[0].unsqueeze(0), torch.tensor([x[0].shape[0]]), None, bert[0].unsqueeze(0), top_k=1,
                                   early_stop_num=0)
    assert tuple(y.shape) == (1, 0) and idx == 0
    ys, idx = net.infer_panel_naive_batched(x, torch.tensor(GOLD["cfg"]["x_lens"]), None, bert, top_k=1, early_stop_num=0)
    assert idx == [0] * len(x) and all(tuple(t.shape) == (0,) for t in ys)
