#!/usr/bin/env python
"""Pin the prompt-free decoding oracle (oracle/gpt_ref_free_oracle.py infer_panel_ref_free) against the reference's unmodified
Text2SemanticDecoder.infer_panel_naive_batched(x, x_lens, None, bert, ...) (t2s_model.py:732-863) on the CPU and write
tests/golden/infer_ref_free.json.

Greedy (top_k = 1, repetition penalty 1.35), B = 4 rows with ragged text lengths, 3 layers, no prompt.  The EOS row of
ar_predict_layer is scaled so that at least one row ends on EOS (which the first 11 steps exclude), at least one reaches
early_stop_num, and some row has EOS as the argmax of its raw logits inside the 11-step window (so the window changes a result;
the golden and the report record it).  Tokens must be identical, per-step logits equal to fp32 noise.

Usage:  EVK_REFERENCE=<reference checkout> python oracle/pin_infer_ref_free.py
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gpt_oracle, gpt_ref_free_oracle  # noqa: E402
from oracle.pin_against_reference import GOLD, import_reference, maxdiff, stub_torchmetrics  # noqa: E402

CFG = dict(n_layer=3, param_seed=14, seed=41, B=4, x_lens=[21, 13, 17, 9], early_stop_num=30, top_k=1, repetition_penalty=1.35,
           temperature=1.0, eos_scale=None)
EOS_SCALES = [1.0, 1.1, 1.2, 1.3, 1.4, 1.5, 1.6, 1.8, 2.0, 2.2, 2.5]
EOS_WINDOW = 11                          # t2s_model.py:835-836
LOGIT_IDS = list(range(0, 1025, 16))     # the classes whose logits the golden keeps (every 16th, EOS included), to 6 decimals


def inputs(cfg, m):
    g = torch.Generator().manual_seed(cfg["seed"])
    x = [torch.randint(0, m["phoneme_vocab_size"], (n,), generator=g) for n in cfg["x_lens"]]
    bert = [torch.randn(1024, n, generator=g) for n in cfg["x_lens"]]
    return x, bert


def params(cfg, m):
    P = gpt_oracle.init_params(gpt_oracle.gpt_param_spec(m), cfg["param_seed"])
    P["ar_text_position.alpha"].fill_(0.8); P["ar_audio_position.alpha"].fill_(1.3)
    P["ar_predict_layer.weight"][m["EOS"]] *= cfg["eos_scale"]
    return P


def run_oracle(cfg, m, trace=None):
    x, bert = inputs(cfg, m)
    return gpt_ref_free_oracle.infer_panel_ref_free(params(cfg, m), x, bert, top_k=cfg["top_k"], early_stop_num=cfg["early_stop_num"],
                                                    temperature=cfg["temperature"], repetition_penalty=cfg["repetition_penalty"], m=m,
                                                    trace=trace)


def pin_infer_ref_free():
    stub_torchmetrics()
    import src.easevoice.soundstorm.auto_reg.models.t2s_model as t2s_mod
    m = dict(gpt_oracle.GPT_MODEL, n_layer=CFG["n_layer"])
    cfg = dict(CFG)
    E = cfg["early_stop_num"]
    for s in EOS_SCALES:                 # the smallest scale with a row ending on EOS, a row reaching early stop, and a row whose
        cfg["eos_scale"] = s             # raw argmax is EOS inside the window (so the window changes a result)
        tr = []
        y, _ = run_oracle(cfg, m, trace=tr)
        n = [len(t) for t in y]
        window = any(int(tr[k][b].argmax()) == m["EOS"] for b in range(cfg["B"]) for k in range(min(EOS_WINDOW, n[b] + 1)))
        if any(EOS_WINDOW <= v < E for v in n) and any(v == E for v in n) and window:
            break
    else:
        raise SystemExit(f"no EOS scale in {EOS_SCALES} gives both ways of finishing and an EOS argmax in the window (last lengths {n})")
    tr = []
    y_ora, idx_ora = run_oracle(cfg, m, trace=tr)
    ref = t2s_mod.Text2SemanticDecoder({"model": m}).eval()
    ref.load_state_dict(params(cfg, m))
    x, bert = inputs(cfg, m)
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
            y_ref, idx_ref = ref.infer_panel_naive_batched(x, torch.tensor(cfg["x_lens"]), None, bert, top_k=cfg["top_k"], top_p=100,
                                                           early_stop_num=E, temperature=cfg["temperature"],
                                                           repetition_penalty=cfg["repetition_penalty"])
    finally:
        t2s_mod.sample = orig_sample
    assert list(idx_ref) == [0] * cfg["B"] == list(idx_ora), (idx_ref, idx_ora)
    assert all(torch.equal(a.long(), b.long()) for a, b in zip(y_ref, y_ora)), (y_ref, y_ora)
    # the reference decodes the rows one after another; row b stops at step len(y_b) (its last sample is dropped)
    stop = [len(t) for t in y_ref]
    assert len(seen) == sum(s + 1 for s in stop), (len(seen), stop)
    err, margins, window_eos, k = 0.0, [[] for _ in range(cfg["B"])], False, 0
    for b in range(cfg["B"]):
        for s in range(stop[b] + 1):
            raw, pen = seen[k]
            k += 1
            err = max(err, maxdiff(raw[0], tr[s][b, :raw.shape[1]]))
            t2 = pen[0].topk(2).values
            margins[b].append(float(t2[0] - t2[1]))
            window_eos |= s < EOS_WINDOW and int(tr[s][b].argmax()) == m["EOS"]
    assert err < 2e-4, err
    steps = sorted({0, 1, 5, EOS_WINDOW, max(stop)})
    gold = {"cfg": cfg, "tokens": [t.tolist() for t in y_ref], "stop": stop, "idx": list(idx_ref),
            "top2_margin": [[round(v, 6) for v in r] for r in margins], "logit_ids": LOGIT_IDS, "eos_argmax_in_window": window_eos,
            "logits_step": {str(s): {str(b): [round(float(v), 6) for v in tr[s][b, LOGIT_IDS]] for b in range(cfg["B"]) if stop[b] >= s}
                            for s in steps}}
    with open(os.path.join(GOLD, "infer_ref_free.json"), "w") as f:
        json.dump(gold, f)
    return {"eos_scale": cfg["eos_scale"], "stop": stop, "steps": len(seen), "max_logit_diff_oracle_vs_reference": err,
            "min_top2_margin": min(min(v) for v in margins), "eos_argmax_in_window": window_eos}


if __name__ == "__main__":
    torch.manual_seed(0)
    import_reference()
    print(pin_infer_ref_free())
