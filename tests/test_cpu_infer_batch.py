"""CPU tests of batched AR decoding (Text2SemanticDecoder.infer_panel_batch_infer): the cache-free oracle against the
reference's own results (tests/golden/infer_batch.json, oracle/pin_infer_batch.py) and the host-side argument handling."""
import json
import os

import pytest
import torch

from oracle import gpt_oracle, gpt_batch_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_batch.json")))


def _case(max_len=None, padded=False):
    c = GOLD["cfg"]
    m = dict(gpt_oracle.GPT_MODEL, n_layer=c["n_layer"])
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), c["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][m["EOS"]] *= c["eos_scale"]
    g = torch.Generator().manual_seed(c["seed"])
    x = [torch.randint(0, m["phoneme_vocab_size"], (n,), generator=g) for n in c["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in c["x_lens"]]
    prompts = torch.randint(0, 1024, (1, c["Yp"]), generator=g).expand(c["B"], -1)
    if padded:                            # a padded [B, X] tensor: every row has width X, its bert features zero-padded
        X = max(c["x_lens"])
        xt = torch.zeros(c["B"], X, dtype=torch.long)
        bt = []
        for b, n in enumerate(c["x_lens"]):
            xt[b, :n] = x[b]
            bt.append(torch.nn.functional.pad(bert[b], (0, X - n)))
        x, bert = list(xt), bt
    tr = []
    y, idx = gpt_batch_oracle.infer_panel_batch(P, x, torch.tensor(c["x_lens"]), bert, prompts, top_k=c["top_k"],
                                                early_stop_num=c["early_stop_num"], temperature=c["temperature"],
                                                repetition_penalty=c["repetition_penalty"], max_len=max_len or c["max_len"], m=m, trace=tr)
    return y, idx, tr


def test_oracle_reproduces_reference_golden():
    y, idx, tr = _case()
    assert [t.tolist() for t in y] == GOLD["tokens"]
    assert idx == GOLD["idx"]
    E = GOLD["cfg"]["early_stop_num"]
    assert sum(i == E for i in idx) == len(idx) - 1 and min(idx) < E // 2       # both ways of finishing are covered
    for s, rows in GOLD["logits_step"].items():
        for b, ref in rows.items():
            assert float((tr[int(s)][int(b), GOLD["logit_ids"]] - torch.tensor(ref)).abs().max()) < 2e-4, (s, b)


def test_oracle_does_not_depend_on_padding():
    y0, i0, tr0 = _case()
    for kw in (dict(max_len=GOLD["cfg"]["max_len"] + 6), dict(padded=True)):
        y1, i1, tr1 = _case(**kw)
        assert i1 == i0 and all(torch.equal(a, b) for a, b in zip(y0, y1)), kw
        assert max(float((a - b).abs().max()) for a, b in zip(tr0, tr1)) < 1e-4, kw


def _net():
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    return Text2SemanticDecoder({"model": dict(gpt_oracle.GPT_MODEL, n_layer=2)})


@pytest.mark.parametrize("top_k", [0, -100, 1026, 2.5])
def test_top_k_outside_vocabulary_is_rejected(top_k):
    x = [torch.zeros(5, dtype=torch.long)]
    with pytest.raises(ValueError, match="top_k"):
        _net().infer_panel_batch_infer(x, torch.tensor([5]), torch.zeros(1, 3, dtype=torch.long), [torch.zeros(1024, 5)], top_k=top_k)


def test_mismatched_rows_are_rejected():
    net = _net()
    x = [torch.zeros(5, dtype=torch.long), torch.zeros(4, dtype=torch.long)]
    prompts = torch.zeros(2, 3, dtype=torch.long)
    with pytest.raises(ValueError, match="one entry per row"):
        net.infer_panel_batch_infer(x, torch.tensor([5, 4]), prompts, [torch.zeros(1024, 5)], top_k=5)
    with pytest.raises(ValueError, match="row 1"):              # bert width must equal the row's width
        net.infer_panel_batch_infer(x, torch.tensor([5, 4]), prompts, [torch.zeros(1024, 5), torch.zeros(1024, 5)], top_k=5)
    with pytest.raises(ValueError, match="row 0"):              # a row wider than max_len
        net.infer_panel_batch_infer(x, torch.tensor([5, 4]), prompts, [torch.zeros(1024, 5), torch.zeros(1024, 4)], top_k=5, max_len=4)


def test_prompt_free_call_goes_to_the_naive_loop():
    net = _net()
    calls = []

    def naive(x, x_lens, prompts, bert, top_k, top_p, early_stop_num, temperature, repetition_penalty, **kw):
        calls.append((tuple(x.shape), int(x_lens), prompts, tuple(bert.shape), top_k, top_p, early_stop_num, temperature, repetition_penalty))
        return torch.arange(4).unsqueeze(0), len(calls)
    net.infer_panel_naive = naive
    x = torch.zeros(2, 6, dtype=torch.long)
    y, idx = net.infer_panel_batch_infer(x, torch.tensor([6, 3]), None, [torch.zeros(1024, 6)] * 2, top_k=7, top_p=0.8,
                                         early_stop_num=9, temperature=0.7, repetition_penalty=2.0)
    # t2s_model.py:576-578 does not pass repetition_penalty on: the naive loop runs with its default 1.35
    assert calls == [((1, 6), 6, None, (1, 1024, 6), 7, 0.8, 9, 0.7, 1.35), ((1, 6), 3, None, (1, 1024, 6), 7, 0.8, 9, 0.7, 1.35)]
    assert idx == [1, 2] and all(torch.equal(t, torch.arange(4)) for t in y)
    with pytest.raises(NotImplementedError):                   # and that path has no prompt-free decoding
        _net().infer_panel_batch_infer(x, torch.tensor([6, 3]), None, [torch.zeros(1024, 6)] * 2, top_k=7)
