#!/usr/bin/env python
"""Pin the batched-decoding oracle (oracle/gpt_batch_oracle.py) against the reference's unmodified
Text2SemanticDecoder.infer_panel_batch_infer (t2s_model.py:563-730) on the CPU and write tests/golden/infer_batch.json.

Greedy (top_k = 1, repetition penalty 1.35), B = 4 rows with ragged text lengths and one shared prompt, 3 layers.  The EOS row
of ar_predict_layer is scaled so that one row ends on EOS well before the others and the rest reach early_stop_num: both ways
of finishing are then in the golden.  Tokens and idx must be identical, per-step logits equal to fp32 noise.

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_infer_batch.py
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gpt_oracle, gpt_batch_oracle  # noqa: E402
from oracle.pin_against_reference import GOLD, import_reference, maxdiff, stub_torchmetrics  # noqa: E402

CFG = dict(n_layer=3, param_seed=14, seed=33, B=4, x_lens=[21, 13, 17, 9], max_len=21, Yp=11, early_stop_num=30, top_k=1,
           repetition_penalty=1.35, temperature=1.0, eos_scale=None)
EOS_SCALES = [1.0, 1.1, 1.2, 1.3, 1.4, 1.5, 1.6, 1.8, 2.0]
LOGIT_IDS = list(range(0, 1025, 16))     # the classes whose logits the golden keeps (every 16th, EOS included), to 6 decimals


def inputs(cfg, m):
    g = torch.Generator().manual_seed(cfg["seed"])
    x = [torch.randint(0, m["phoneme_vocab_size"], (n,), generator=g) for n in cfg["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in cfg["x_lens"]]
    prompt = torch.randint(0, 1024, (1, cfg["Yp"]), generator=g)
    return x, bert, prompt.expand(cfg["B"], -1)


def params(cfg, m):
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), cfg["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][m["EOS"]] *= cfg["eos_scale"]
    return P


def run_oracle(cfg, m, trace=None):
    x, bert, prompts = inputs(cfg, m)
    return gpt_batch_oracle.infer_panel_batch(params(cfg, m), x, torch.tensor(cfg["x_lens"]), bert, prompts, top_k=cfg["top_k"],
                                              early_stop_num=cfg["early_stop_num"], temperature=cfg["temperature"],
                                              repetition_penalty=cfg["repetition_penalty"], max_len=cfg["max_len"], m=m, trace=trace)


def pin_infer_batch():
    stub_torchmetrics()
    import src.easevoice.soundstorm.auto_reg.models.t2s_model as t2s_mod
    m = dict(gpt_oracle.GPT_MODEL, n_layer=CFG["n_layer"])
    cfg = dict(CFG)
    E = cfg["early_stop_num"]
    for s in EOS_SCALES:                 # the smallest scale with one row on EOS well before early stop and the others reaching it
        cfg["eos_scale"] = s
        _, idx = run_oracle(cfg, m)
        if sum(i < E // 2 for i in idx) == 1 and sum(i == E for i in idx) == cfg["B"] - 1:
            break
    else:
        raise SystemExit(f"no EOS scale in {EOS_SCALES} gives one early EOS row (last idx {idx})")
    tr = []
    y_ora, idx_ora = run_oracle(cfg, m, trace=tr)
    ref = t2s_mod.Text2SemanticDecoder({"model": m}).eval()
    ref.load_state_dict(params(cfg, m))
    x, bert, prompts = inputs(cfg, m)
    seen = []
    orig_sample = t2s_mod.sample

    def spy(logits, previous_tokens=None, **kw):
        raw = logits.clone()
        out = orig_sample(logits, previous_tokens, **kw)
        seen.append((raw, logits.clone()))              # the reference penalises `logits` in place: (raw, penalised)
        return out
    t2s_mod.sample = spy
    try:
        with torch.no_grad():
            y_ref, idx_ref = ref.infer_panel_batch_infer(x, torch.tensor(cfg["x_lens"]), prompts, bert, top_k=cfg["top_k"], top_p=100,
                                                         early_stop_num=E, temperature=cfg["temperature"],
                                                         repetition_penalty=cfg["repetition_penalty"], max_len=cfg["max_len"])
    finally:
        t2s_mod.sample = orig_sample
    assert list(idx_ref) == list(idx_ora), (idx_ref, idx_ora)
    assert all(torch.equal(a.long(), b.long()) for a, b in zip(y_ref, y_ora)), (y_ref, y_ora)
    # the reference's batch shrinks as rows finish: at step s it holds the rows still running, in their original order
    fin_step = [i + 1 if i < E else i for i in idx_ref]
    err, margins = 0.0, [[] for _ in range(cfg["B"])]
    for s, (raw, pen) in enumerate(seen):
        alive = [b for b in range(cfg["B"]) if fin_step[b] >= s]
        assert len(alive) == raw.shape[0], (s, alive, raw.shape)
        err = max(err, maxdiff(raw, tr[s][alive, :raw.shape[1]]))
        for r, b in enumerate(alive):
            t2 = pen[r].topk(2).values
            margins[b].append(float(t2[0] - t2[1]))
    assert err < 2e-4, err
    steps = (0, 1, 5, max(fin_step))
    gold = {"cfg": cfg, "tokens": [y.tolist() for y in y_ref], "idx": list(idx_ref),
            "top2_margin": [[round(v, 6) for v in r] for r in margins], "logit_ids": LOGIT_IDS,
            "logits_step": {str(s): {str(b): [round(float(v), 6) for v in tr[s][b, LOGIT_IDS]] for b in range(cfg["B"]) if fin_step[b] >= s}
                            for s in steps}}
    with open(os.path.join(GOLD, "infer_batch.json"), "w") as f:
        json.dump(gold, f)
    return {"eos_scale": cfg["eos_scale"], "idx": list(idx_ref), "steps": len(seen), "max_logit_diff_oracle_vs_reference": err,
            "min_top2_margin": min(min(v) for v in margins)}


if __name__ == "__main__":
    torch.manual_seed(0)
    import_reference()
    print(pin_infer_batch())
