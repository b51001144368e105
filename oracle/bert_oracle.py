"""CPU restatement of the BERT text feature `Normalize.text` and the TTS text front end compute (reference
src/normalization/normalize.py:88-106 `_get_bert_feature`, src/easevoice/inference/preprocessor.py:180-193 `get_bert_feature`):
`bert_model(**tokenizer(text), output_hidden_states=True)["hidden_states"][-3:-2]`, rows 1..-1, each repeated word2ph[i] times,
transposed to [hidden, sum(word2ph)].

TEST INFRASTRUCTURE ONLY (tests/, bench CPU arms).  The model is a third-party dependency of the reference, `transformers`
(this image: 5.5.0; `BertForMaskedLM`, models/bert/modeling_bert.py); the architecture is the published BERT one, restated from
that file's forward passes:

  embeddings  LayerNorm(word[id] + type[tt] + pos[t]), eps 1e-12                             BertEmbeddings
  encoder     post-LN blocks: h = LN(h + O(MHA(h))), h = LN(h + W2 gelu(W1 h)), exact-erf GELU  BertLayer
              MHA: heads x 64, scores scaled by 64^-0.5, keys where attention_mask == 0 excluded

Pinned against `transformers.BertForMaskedLM` itself by oracle/pin_bert.py (golden tests/golden/bert.pt)."""
import math

import torch
import torch.nn.functional as F

BERT_LARGE = dict(vocab_size=21128, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
                  max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)


def param_spec(cfg=BERT_LARGE):
    """state_dict contract of transformers.BertModel (5.5.0) without the pooler (BertForMaskedLM builds it without one)."""
    H, F_ = cfg["hidden_size"], cfg["intermediate_size"]
    s = {"embeddings.word_embeddings.weight": (cfg["vocab_size"], H),
         "embeddings.position_embeddings.weight": (cfg["max_position_embeddings"], H),
         "embeddings.token_type_embeddings.weight": (cfg["type_vocab_size"], H),
         "embeddings.LayerNorm.weight": (H,), "embeddings.LayerNorm.bias": (H,)}
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            s[p + f"attention.self.{n}.weight"] = (H, H)
            s[p + f"attention.self.{n}.bias"] = (H,)
        s[p + "attention.output.dense.weight"] = (H, H)
        s[p + "attention.output.dense.bias"] = (H,)
        s[p + "attention.output.LayerNorm.weight"] = (H,)
        s[p + "attention.output.LayerNorm.bias"] = (H,)
        s[p + "intermediate.dense.weight"] = (F_, H)
        s[p + "intermediate.dense.bias"] = (F_,)
        s[p + "output.dense.weight"] = (H, F_)
        s[p + "output.dense.bias"] = (H,)
        s[p + "output.LayerNorm.weight"] = (H,)
        s[p + "output.LayerNorm.bias"] = (H,)
    return s


def init_params(spec, seed):
    """Seeded synthetic weights (there is no checkpoint offline): fan-in scaled normal matrices, unit-scale embedding rows,
    LayerNorm gains near 1 and non-zero biases everywhere (transformers' own init zeroes the biases, which would hide a bias
    that is dropped or misplaced)."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for k, shp in spec.items():
        if k.endswith("LayerNorm.weight"):
            P[k] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith("bias"):
            P[k] = 0.05 * torch.randn(shp, generator=g)
        elif k.startswith("embeddings."):
            P[k] = 0.5 * torch.randn(shp, generator=g)
        else:
            P[k] = torch.randn(shp, generator=g) / math.sqrt(shp[1])
    return P


def n_layers_run(cfg, index):
    """hidden_states[index] of an L-layer model is the output after this many encoder layers."""
    L = cfg["num_hidden_layers"]
    n = index if index >= 0 else L + 1 + index
    assert 0 <= n <= L, (index, L)
    return n


@torch.no_grad()
def forward(P, cfg, input_ids, attention_mask=None, token_type_ids=None, index=-3):
    """input_ids int64 [B, T] -> hidden_states[index] [B, T, H] (fp32, CPU)."""
    B, T = input_ids.shape
    H, nh, eps = cfg["hidden_size"], cfg["num_attention_heads"], cfg["layer_norm_eps"]
    dh = H // nh
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    x = P["embeddings.word_embeddings.weight"][input_ids] + P["embeddings.token_type_embeddings.weight"][token_type_ids]
    x = x + P["embeddings.position_embeddings.weight"][:T]
    x = F.layer_norm(x, (H,), P["embeddings.LayerNorm.weight"], P["embeddings.LayerNorm.bias"], eps)
    bias = None
    if attention_mask is not None:
        bias = torch.zeros(B, 1, 1, T).masked_fill(attention_mask[:, None, None, :] == 0, float("-inf"))
    for i in range(n_layers_run(cfg, index)):
        p = f"encoder.layer.{i}."

        def lin(t, n):
            return F.linear(t, P[p + n + ".weight"], P[p + n + ".bias"])

        q, k, v = (lin(x, f"attention.self.{n}").view(B, T, nh, dh).transpose(1, 2) for n in ("query", "key", "value"))
        s = (q @ k.transpose(-1, -2)) * (dh ** -0.5)
        if bias is not None:
            s = s + bias
        a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, T, H)
        x = F.layer_norm(lin(a, "attention.output.dense") + x, (H,), P[p + "attention.output.LayerNorm.weight"],
                         P[p + "attention.output.LayerNorm.bias"], eps)
        f = lin(F.gelu(lin(x, "intermediate.dense")), "output.dense")
        x = F.layer_norm(f + x, (H,), P[p + "output.LayerNorm.weight"], P[p + "output.LayerNorm.bias"], eps)
    return x


def phone_level(hidden, word2ph):
    """hidden [T, H] of one sentence -> [H, sum(word2ph)]: character i takes token i + 1, repeated word2ph[i] times
    (normalize.py:99-105)."""
    return torch.cat([hidden[i + 1].repeat(w, 1) for i, w in enumerate(word2ph)], dim=0).T
