"""Oracle (test infrastructure): prompt-free AR decoding of the stage-1 GPT, functional torch fp32, no KV cache.

Restates src/easevoice/soundstorm/auto_reg/models/t2s_model.py `Text2SemanticDecoder.infer_panel_naive_batched` with
prompts None (:732-863: infer_panel_naive on each row in turn) for all rows at once, in the manner of
oracle/gpt_batch_oracle.py: every step re-runs the stack on the whole padded sequence under the prefix-LM mask.
"""
import math

import torch
import torch.nn.functional as F

from oracle.gpt_oracle import GPT_MODEL, logits_to_probs, prefix_lm_mask, sine_pe


def infer_panel_ref_free(P, x, bert, top_k=1, top_p=100, early_stop_num=-1, temperature=1.0, repetition_penalty=1.35, max_len=None,
                         m=GPT_MODEL, draws=None, trace=None, max_steps=1500):
    """Prompt-free decoding (t2s_model.py:732-863 with prompts None: infer_panel_naive on each row in turn), all rows at once.
    Row b's text is all of x[b] (x_lens is not read by the reference's loop); rows are right-padded to max_len (default: the
    longest), and padded text positions are neither attended nor used.  Step idx re-runs the stack on [B, max_len + idx]:
    text attends its row's text, generated token t (embedded at pe[t]) attends its row's text and tokens <= t.  Step 0's logits
    come from each row's last text position, later ones from the last token.  EOS is excluded for idx < 11; a row stops when its
    sample or the argmax of its penalised logits is EOS, or at idx + 1 > early_stop_num, or at idx == max_steps - 1, and then
    keeps the tokens before that step's sample.  draws / trace as in infer_panel_batch.  -> (y_list, [0] * B)."""
    assert draws is not None or top_k == 1, "without supplied draws only greedy decoding is deterministic"
    D, H = m["hidden_dim"], m["head"]
    dk, EOS = D // H, m["EOS"]
    B = len(x)
    lens = torch.tensor([int(t.shape[0]) for t in x])
    max_len = int(max_len if max_len is not None else lens.max())
    pe = sine_pe(max(max_len, max_steps + 2), D)
    xe = torch.zeros(B, max_len, D)
    for b in range(B):
        t = F.embedding(x[b].long(), P["ar_text_embedding.word_embeddings.weight"]) + F.linear(bert[b].t(), P["bert_proj.weight"], P["bert_proj.bias"])
        xe[b, :t.shape[0]] = t + P["ar_text_position.alpha"] * pe[:t.shape[0]]
    y = torch.zeros(B, 0, dtype=torch.long)
    y_list = [None] * B
    for idx in range(max_steps):
        Y = y.shape[1]
        ye = F.embedding(y, P["ar_audio_embedding.word_embeddings.weight"]) + P["ar_audio_position.alpha"] * pe[:Y]
        h = torch.cat([xe, ye], 1)
        mask = prefix_lm_mask(lens, torch.full((B,), Y), max_len, Y)
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
        last = h[torch.arange(B), lens - 1] if Y == 0 else h[:, -1]
        logits = F.linear(last, P["ar_predict_layer.weight"])
        if trace is not None:
            trace.append(logits.clone())
        if idx < 11:
            logits = logits[:, :-1]
        toks = torch.zeros(B, 1, dtype=torch.long)
        for b in range(B):
            if y_list[b] is not None:
                continue
            lb = logits[b:b + 1].clone()
            probs = logits_to_probs(lb, y[b:b + 1], temperature=temperature, top_k=top_k, top_p=top_p,
                                    repetition_penalty=repetition_penalty)
            qd = draws(b, idx, probs.shape[1]).reshape(1, -1) if draws is not None else torch.ones_like(probs)
            toks[b, 0] = int(torch.argmax(probs / qd, dim=-1))
            if (int(toks[b, 0]) == EOS or int(torch.argmax(lb, dim=-1)) == EOS or (early_stop_num != -1 and idx + 1 > early_stop_num)
                    or idx == max_steps - 1):
                y_list[b] = y[b].clone()
        y = torch.cat([y, toks], 1)
        if None not in y_list:
            break
    return y_list, [0] * B
