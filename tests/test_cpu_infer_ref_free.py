"""CPU tests of prompt-free AR decoding (Text2SemanticDecoder.infer_panel_naive_batched with prompts None): the cache-free oracle
against the reference's own results (tests/golden/infer_ref_free.json, oracle/pin_infer_ref_free.py) and the host-side argument
handling."""
import json
import os

import pytest
import torch

from oracle import gpt_oracle, gpt_ref_free_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "infer_ref_free.json")))


def _case(max_len=None):
    c = GOLD["cfg"]
    m = dict(gpt_oracle.GPT_MODEL, n_layer=c["n_layer"])
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), c["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][m["EOS"]] *= c["eos_scale"]
    g = torch.Generator().manual_seed(c["seed"])
    x = [torch.randint(0, m["phoneme_vocab_size"], (n,), generator=g) for n in c["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in c["x_lens"]]
    tr = []
    y, idx = gpt_ref_free_oracle.infer_panel_ref_free(P, x, bert, top_k=c["top_k"], early_stop_num=c["early_stop_num"],
                                                      temperature=c["temperature"], repetition_penalty=c["repetition_penalty"],
                                                      max_len=max_len, m=m, trace=tr)
    return y, idx, tr


def test_oracle_reproduces_reference_golden():
    y, idx, tr = _case()
    assert [t.tolist() for t in y] == GOLD["tokens"]
    assert idx == GOLD["idx"] == [0] * len(y)
    assert [len(t) for t in y] == GOLD["stop"]
    E = GOLD["cfg"]["early_stop_num"]
    # both ways of finishing are covered, and the 11-step EOS window changed a result
    assert E in GOLD["stop"] and any(11 <= s < E for s in GOLD["stop"]) and GOLD["eos_argmax_in_window"]
    for s, rows in GOLD["logits_step"].items():
        for b, ref in rows.items():
            assert float((tr[int(s)][int(b), GOLD["logit_ids"]] - torch.tensor(ref)).abs().max()) < 2e-4, (s, b)


def test_oracle_does_not_depend_on_padding():
    y0, i0, tr0 = _case()
    y1, i1, tr1 = _case(max_len=max(GOLD["cfg"]["x_lens"]) + 6)
    assert i1 == i0 and all(torch.equal(a, b) for a, b in zip(y0, y1))
    assert max(float((a - b).abs().max()) for a, b in zip(tr0, tr1)) < 1e-4


def _net():
    from easevoice_trainer_b200.models_gpt import Text2SemanticDecoder
    return Text2SemanticDecoder({"model": dict(gpt_oracle.GPT_MODEL, n_layer=2)})


@pytest.mark.parametrize("top_k", [0, -100, 1026, 2.5])
def test_top_k_outside_vocabulary_is_rejected(top_k):
    x = [torch.zeros(5, dtype=torch.long)]
    with pytest.raises(ValueError, match="top_k"):
        _net().infer_panel_naive_batched(x, torch.tensor([5]), None, [torch.zeros(1024, 5)], top_k=top_k)
    with pytest.raises(ValueError, match="top_k"):              # through infer_panel_batch_infer's forwarding as well
        _net().infer_panel_batch_infer(x, torch.tensor([5]), None, [torch.zeros(1024, 5)], top_k=top_k)


def test_mismatched_rows_are_rejected():
    net = _net()
    x = [torch.zeros(5, dtype=torch.long), torch.zeros(4, dtype=torch.long)]
    with pytest.raises(ValueError, match="one entry per row"):
        net.infer_panel_naive_batched(x, torch.tensor([5, 4]), None, [torch.zeros(1024, 5)], top_k=5)
    with pytest.raises(ValueError, match="row 1"):              # bert width must equal the row's width
        net.infer_panel_naive_batched(x, torch.tensor([5, 4]), None, [torch.zeros(1024, 5), torch.zeros(1024, 5)], top_k=5)
    with pytest.raises(ValueError, match="row 0"):              # x_lens is not read: a padded row's bert must have its full width
        net.infer_panel_naive_batched(torch.zeros(2, 6, dtype=torch.long), torch.tensor([5, 4]), None,
                                      [torch.zeros(1024, 5), torch.zeros(1024, 4)], top_k=5)


def test_cpu_inputs_have_no_prompt_free_path():
    x = [torch.zeros(5, dtype=torch.long)]
    with pytest.raises(NotImplementedError):
        _net().infer_panel_naive(x[0].unsqueeze(0), torch.tensor([5]), None, torch.zeros(1, 1024, 5), top_k=5)
    with pytest.raises(NotImplementedError):                   # with a prompt there is no CPU path either
        _net().infer_panel_naive(x[0].unsqueeze(0), torch.tensor([5]), torch.zeros(1, 3, dtype=torch.long), torch.zeros(1, 1024, 5),
                                 top_k=5)
    with pytest.raises(NotImplementedError):
        _net().infer_panel_naive_batched(x, torch.tensor([5]), None, [torch.zeros(1024, 5)], top_k=5)
