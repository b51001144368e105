"""Float64 restatement of the stage-1 GPT's AR decoding under a 16-bit compute type (Text2SemanticDecoder.set_compute_type),
with the contract's rounding points: both operands of every Linear -- bert_proj, in_proj, out_proj, linear1, linear2 and the
head -- rounded to nearest even to 16 bits (the activation from its fp32 value, the weight from the fp32 parameter), then
multiplied and summed in float64; the K and V of every position rounded the same way as they enter the cache.  The prompt
pass attends the unrounded qkv; a token step attends the rounded cache with its unrounded q.  Everything else is
oracle/gpt_oracle.py's float64 computation.  One row without padding: the decoder never attends a row's padding, so padding
does not change its values.  dtype None rounds nothing (the fp32 decoder's computation, in float64)."""
import math

import torch
import torch.nn.functional as F

from oracle import gpt_oracle as O


def h16(x, dtype):
    """x rounded to fp32, then to nearest even in `dtype` (torch.float16 / torch.bfloat16), as float64; dtype None: x."""
    return x.double() if dtype is None else x.float().to(dtype).double()


LINEARS = ("bert_proj.weight", "self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight",
           "ar_predict_layer.weight")


def rounded(P, dtype):
    """The parameters in float64, every Linear's weight rounded once to `dtype` (as ops.pack_weight_h16 packs it)."""
    return {k: h16(v, dtype) if k.endswith(LINEARS) else v.double() for k, v in P.items()}


def lin(x, w, b, dtype):
    """h(x) w^T + b, w already rounded (rounded())."""
    y = h16(x, dtype) @ w.T
    return y if b is None else y + b


def _ffn(P, p, h, a, dtype):
    """the block after its attention output a: out_proj, residual + LayerNorm, linear1 + ReLU, linear2, residual + LayerNorm"""
    D = h.shape[-1]
    h = F.layer_norm(h + lin(a, P[p + "self_attn.out_proj.weight"], P[p + "self_attn.out_proj.bias"], dtype), (D,),
                     P[p + "norm1.weight"], P[p + "norm1.bias"], 1e-5)
    f = lin(torch.relu(lin(h, P[p + "linear1.weight"], P[p + "linear1.bias"], dtype)), P[p + "linear2.weight"], P[p + "linear2.bias"], dtype)
    return F.layer_norm(h + f, (D,), P[p + "norm2.weight"], P[p + "norm2.bias"], 1e-5)


def _attend(q, k, v, H, mask=None):
    """q [T, D], k / v [S, D] -> [T, D]; mask [T, S] True = masked."""
    T, D = q.shape
    qh, kh, vh = (t.view(t.shape[0], H, D // H).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / math.sqrt(D // H)
    if mask is not None:
        s = s.masked_fill(mask, float("-inf"))
    return (s.softmax(-1) @ vh).transpose(0, 1).reshape(T, D)


class Decoder:
    """Incremental decoding of one row, as the decoder runs it: prompt() is the prompt pass, step(token) one token step."""

    def __init__(self, P, m, dtype):
        self.P = rounded(P, dtype)
        self.m, self.dtype = m, dtype
        self.pe = None

    def prompt(self, x, bert, prompt=None):
        """x [X] phoneme ids, bert [1024, X], prompt [Yp] semantic tokens or None -> the first logits [V]: from the last prompt
        position with a prompt, from the last text position without.  Fills the K/V caches."""
        P, m, dt = self.P, self.m, self.dtype
        D, H = m["hidden_dim"], m["head"]
        X, Yp = x.shape[0], 0 if prompt is None else prompt.shape[0]
        self.Yp, self.steps = Yp, 0
        self.pe = O.sine_pe(max(X, Yp) + 2048, D).double()
        xe = P["ar_text_embedding.word_embeddings.weight"][x] + lin(bert.T, P["bert_proj.weight"], P["bert_proj.bias"], dt)
        h = xe + P["ar_text_position.alpha"] * self.pe[:X]
        if Yp:
            ye = P["ar_audio_embedding.word_embeddings.weight"][prompt] + P["ar_audio_position.alpha"] * self.pe[:Yp]
            h = torch.cat([h, ye])
        mask = O.prefix_lm_mask(torch.tensor([X]), torch.tensor([Yp]), X, Yp)[0]
        self.K, self.V = [], []
        for i in range(m["n_layer"]):
            p = f"h.layers.{i}."
            qkv = lin(h, P[p + "self_attn.in_proj_weight"], P[p + "self_attn.in_proj_bias"], dt)
            q, k, v = qkv.split(D, -1)
            self.K.append(h16(k, dt))
            self.V.append(h16(v, dt))
            h = _ffn(P, p, h, _attend(q, k, v, H, mask), dt)
        return lin(h[-1:], P["ar_predict_layer.weight"], None, dt)[0]

    def step(self, token):
        """The token sampled at step idx, embedded at pe[Yp + idx], its K and V rounded into the caches -> the next logits [V]."""
        P, m, dt = self.P, self.m, self.dtype
        D, H = m["hidden_dim"], m["head"]
        h = (P["ar_audio_embedding.word_embeddings.weight"][int(token)] + P["ar_audio_position.alpha"] * self.pe[self.Yp + self.steps])[None]
        for i in range(m["n_layer"]):
            p = f"h.layers.{i}."
            q, k, v = lin(h, P[p + "self_attn.in_proj_weight"], P[p + "self_attn.in_proj_bias"], dt).split(D, -1)
            self.K[i] = torch.cat([self.K[i], h16(k, dt)])
            self.V[i] = torch.cat([self.V[i], h16(v, dt)])
            h = _ffn(P, p, h, _attend(q, self.K[i], self.V[i], H), dt)
        self.steps += 1
        return lin(h, P["ar_predict_layer.weight"], None, dt)[0]


def teacher_forced(P, m, dtype, x, bert, prompt, tokens):
    """-> [1 + len(tokens), V]: the first logits, then the logits after each of `tokens` (the decoder's trace)."""
    dec = Decoder(P, m, dtype)
    out = [dec.prompt(x, bert, prompt)]
    out += [dec.step(t) for t in tokens]
    return torch.stack(out)


def penalised(logits, history, penalty):
    """utils.py:121-125 on one row: the logits of the tokens in `history` divided by the penalty (multiplied when negative)."""
    out = logits.clone()
    idx = torch.tensor(sorted(set(int(t) for t in history)), dtype=torch.long)
    if len(idx) and penalty != 1.0:
        s = out[idx]
        out[idx] = torch.where(s < 0, s * penalty, s / penalty)
    return out
