"""Oracle (test infrastructure): batched AR decoding of the stage-1 GPT, functional torch fp32, no KV cache.

Restates src/easevoice/soundstorm/auto_reg/models/t2s_model.py `Text2SemanticDecoder.infer_panel_batch_infer` (:563-730):
every step re-runs the stack on the whole padded sequence [B, max_len + Y] under the reference's mask (text rows right-padded
to max_len; padded text positions are never attended; audio rows see their row's text and earlier audio), which is what
process_prompt + decode_next_token compute incrementally.  Retirement and `idx` rules as in the reference:
  - EOS excluded at step 0 only;
  - a row stops when its sampled token or the argmax of its penalised logits is EOS -> (y[:-1], idx - 1);
  - at early_stop_num (idx + 1 > early_stop_num) or idx == 1499 every remaining row stops -> (y[:-1], idx).
Finished rows stay in the batch here (the reference removes them); rows are independent, so the results are the same.
"""
import math

import torch
import torch.nn.functional as F

from oracle.gpt_oracle import GPT_MODEL, logits_to_probs, prefix_lm_mask, sine_pe


def infer_panel_batch(P, x, x_lens, bert, prompts, top_k=1, top_p=100, early_stop_num=-1, temperature=1.0, repetition_penalty=1.35,
                      max_len=None, m=GPT_MODEL, draws=None, trace=None, max_steps=1500):
    """x: list of 1-D phoneme ids; bert: list of [1024, X_b]; x_lens [B]; prompts [B, Yp].
    draws(b, idx, n) -> the Exp(1) draws [n] of row b at step idx (None: greedy, top_k = 1 needed).
    trace (list) receives the raw [B, V] logits of every step.  -> (y_list, idx_list)."""
    assert draws is not None or top_k == 1, "without supplied draws only greedy decoding is deterministic"
    D, H = m["hidden_dim"], m["head"]
    dk, EOS = D // H, m["EOS"]
    B, Yp = prompts.shape
    x_lens = torch.as_tensor(x_lens).long()
    max_len = int(max_len if max_len is not None else x_lens.max())
    pe = sine_pe(max(max_len, Yp + max_steps + 2), D)
    xe = torch.zeros(B, max_len, D)
    for b in range(B):                    # :581-589: embedded, positioned, then zero-padded to max_len
        t = F.embedding(x[b].long(), P["ar_text_embedding.word_embeddings.weight"]) + F.linear(bert[b].t(), P["bert_proj.weight"], P["bert_proj.bias"])
        xe[b, :t.shape[0]] = t + P["ar_text_position.alpha"] * pe[:t.shape[0]]
    y = prompts.long().clone()
    y_list, idx_list = [None] * B, [None] * B
    for idx in range(max_steps):
        Y = y.shape[1]
        ye = F.embedding(y, P["ar_audio_embedding.word_embeddings.weight"]) + P["ar_audio_position.alpha"] * pe[:Y]
        h = torch.cat([xe, ye], 1)
        mask = prefix_lm_mask(x_lens, torch.full((B,), Y), max_len, Y)
        add = torch.zeros(mask.shape).masked_fill(mask, float("-inf")).unsqueeze(1)
        L = max_len + Y
        for i in range(m["n_layer"]):
            p = f"h.layers.{i}."
            qkv = F.linear(h, P[p + "self_attn.in_proj_weight"], P[p + "self_attn.in_proj_bias"])
            q, k, v = [t.view(B, L, H, dk).transpose(1, 2) for t in qkv.split(D, dim=-1)]
            att = torch.softmax(q @ k.transpose(-2, -1) / math.sqrt(dk) + add, dim=-1) @ v
            att = F.linear(att.transpose(1, 2).reshape(B, L, D), P[p + "self_attn.out_proj.weight"], P[p + "self_attn.out_proj.bias"])
            h = F.layer_norm(h + att, (D,), P[p + "norm1.weight"], P[p + "norm1.bias"], 1e-5)
            ff = F.linear(torch.relu(F.linear(h, P[p + "linear1.weight"], P[p + "linear1.bias"])), P[p + "linear2.weight"], P[p + "linear2.bias"])
            h = F.layer_norm(h + ff, (D,), P[p + "norm2.weight"], P[p + "norm2.bias"], 1e-5)
        logits = F.linear(h[:, -1], P["ar_predict_layer.weight"])
        if trace is not None:
            trace.append(logits.clone())
        if idx == 0:
            logits = logits[:, :-1]
        toks = torch.zeros(B, 1, dtype=torch.long)
        for b in range(B):
            if idx_list[b] is not None:
                continue
            lb = logits[b:b + 1].clone()
            probs = logits_to_probs(lb, y[b:b + 1], temperature=temperature, top_k=top_k, top_p=top_p,
                                    repetition_penalty=repetition_penalty)
            qd = draws(b, idx, probs.shape[1]).reshape(1, -1) if draws is not None else torch.ones_like(probs)
            toks[b, 0] = int(torch.argmax(probs / qd, dim=-1))
            if int(toks[b, 0]) == EOS or int(torch.argmax(lb, dim=-1)) == EOS:      # lb carries the in-place penalty
                idx_list[b], y_list[b] = idx - 1, torch.cat([y[b], toks[b]])[:-1]
        y = torch.cat([y, toks], 1)
        if (early_stop_num != -1 and idx + 1 > early_stop_num) or idx == max_steps - 1:
            for b in range(B):
                if idx_list[b] is None:
                    idx_list[b], y_list[b] = idx, y[b, :-1].clone()
        if None not in idx_list:
            break
    return y_list, idx_list
