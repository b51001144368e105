"""BERT text features of the dataset preparation step (SURVEY section 8 row f3, text half) and of the TTS text front end.

`Normalize._get_bert_feature` (reference src/normalization/normalize.py:88-106) and `TextPreprocessor.get_bert_feature`
(src/easevoice/inference/preprocessor.py:180-193) both compute

    inputs = tokenizer(norm_text, return_tensors="pt")                                  # [CLS] ... [SEP]
    res = bert_model(**inputs, output_hidden_states=True)["hidden_states"][-3:-2]     # after L - 2 of L encoder layers
    feature[:, phones of character i] = res[0][i + 1]  (repeated word2ph[i] times)  -> [hidden, sum(word2ph)] fp32

with `chinese-roberta-wwm-ext-large` (transformers `BertForMaskedLM`, 24 layers, 1024 wide).  This module is that computation
on the library's kernels, with the same state_dict keys:

  embeddings  evk_embedding row gathers (word, token type, position) + the residual LayerNorm kernel, eps 1e-12
  encoder     post-LN blocks: one packed QKV Linear, fused padded attention (evk_attn_pad_fwd, head dim 64), output Linear +
              residual LayerNorm, Linear + exact-erf GELU + Linear + residual LayerNorm
  phones      host-built row index map -> evk_embedding gather, row mask, evk_transpose_bct_btc to channel-first

Only the layers that `hidden_states[index]` depends on run; the last two layers and the MLM head never do.  Several
utterances run in one right-padded batch: keys past a row's length are excluded, so every valid row equals that utterance
run alone.  Inference only, fp32 storage, TF32 tensor-core products like the rest of the library.  No CPU fallback; every check
on the inputs happens before the first library call.
"""
import json
import os

import torch

from . import ops
from .models import ParamTree
from .normalize_token import format_path

BERT_LARGE = dict(vocab_size=21128, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
                  max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act="gelu",
                  position_embedding_type="absolute")
HEAD_DIM = 64          # the fused attention kernel's head dim


class BertModel(ParamTree):
    """transformers.BertModel (modeling_bert.py) without the pooler, as `BertForMaskedLM.bert` holds it."""

    def __init__(self, config=None):
        super().__init__()
        c = dict(BERT_LARGE, **(config or {}))
        if c["hidden_act"] != "gelu":
            raise ValueError(f"hidden_act {c['hidden_act']!r} unsupported (exact-erf 'gelu' only)")
        if c["position_embedding_type"] != "absolute":
            raise ValueError(f"position_embedding_type {c['position_embedding_type']!r} unsupported ('absolute' only)")
        if c["hidden_size"] != c["num_attention_heads"] * HEAD_DIM:
            raise ValueError(f"hidden_size {c['hidden_size']} != {c['num_attention_heads']} heads x {HEAD_DIM}")
        self.cfg = c
        H, F, P = c["hidden_size"], c["intermediate_size"], "encoder.layer."
        self._register("embeddings.word_embeddings.weight", torch.zeros(c["vocab_size"], H))
        self._register("embeddings.position_embeddings.weight", torch.zeros(c["max_position_embeddings"], H))
        self._register("embeddings.token_type_embeddings.weight", torch.zeros(c["type_vocab_size"], H))
        self._register("embeddings.LayerNorm.weight", torch.ones(H))
        self._register("embeddings.LayerNorm.bias", torch.zeros(H))
        for i in range(c["num_hidden_layers"]):
            p = f"{P}{i}."
            for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
                self._register(p + n + ".weight", torch.zeros(H, H))
                self._register(p + n + ".bias", torch.zeros(H))
            self._register(p + "intermediate.dense.weight", torch.zeros(F, H))
            self._register(p + "intermediate.dense.bias", torch.zeros(F))
            self._register(p + "output.dense.weight", torch.zeros(H, F))
            self._register(p + "output.dense.bias", torch.zeros(H))
            for n in ("attention.output.LayerNorm", "output.LayerNorm"):
                self._register(p + n + ".weight", torch.ones(H))
                self._register(p + n + ".bias", torch.zeros(H))

    # ---- loading ----------------------------------------------------------------------------------------------------------
    @staticmethod
    def map_state_dict(sd):
        """BertForMaskedLM / BertModel checkpoint keys -> this module's: the `bert.` prefix is accepted, the MLM head (`cls.*`),
        the pooler and the `position_ids` buffers are dropped, and the old LayerNorm `gamma` / `beta` names map to
        `weight` / `bias`."""
        out = {}
        for k, t in sd.items():
            if k.startswith("bert."):
                k = k[len("bert."):]
            if k.startswith("cls.") or k.startswith("pooler.") or k.endswith(".position_ids"):
                continue
            if k.endswith("LayerNorm.gamma"):
                k = k[:-len("gamma")] + "weight"
            elif k.endswith("LayerNorm.beta"):
                k = k[:-len("beta")] + "bias"
            out[k] = t.float()
        return out

    def load_state_dict(self, sd, strict=True):
        return super().load_state_dict(self.map_state_dict(sd), strict=strict)

    @classmethod
    def from_pretrained(cls, base_path, device="cuda"):
        """`AutoModelForMaskedLM.from_pretrained(base_path)` for a local directory with config.json and pytorch_model.bin (or
        model.safetensors when the `safetensors` package is importable); the MLM head is not loaded."""
        if not os.path.exists(base_path):
            raise FileNotFoundError(base_path)
        cfg = {}
        cj = os.path.join(base_path, "config.json")
        if os.path.exists(cj):
            with open(cj) as f:
                raw = json.load(f)
            cfg = {k: raw[k] for k in BERT_LARGE if k in raw}
        net = cls(cfg)
        pt, st = os.path.join(base_path, "pytorch_model.bin"), os.path.join(base_path, "model.safetensors")
        if os.path.exists(pt):
            sd = torch.load(pt, map_location="cpu", weights_only=False)
        elif os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            raise FileNotFoundError(f"no pytorch_model.bin / model.safetensors under {base_path}")
        net.load_state_dict(sd, strict=True)
        return net.to(device).eval()

    # ---- forward ------------------------------------------------------------------------------------------------------------
    def layers_for(self, index):
        """hidden_states[index] is the output after this many encoder layers (hidden_states[0] is the embedding output)."""
        L = self.cfg["num_hidden_layers"]
        n = index if index >= 0 else L + 1 + index
        if not 0 <= n <= L:
            raise ValueError(f"hidden state index {index} out of range for {L} layers")
        return n

    def check_inputs(self, input_ids, attention_mask=None, token_type_ids=None):
        """-> (ids, token types, lengths), int64 CPU [B, T], [B, T] and [B].  Raises ValueError on anything the forward cannot
        take: more than max_position_embeddings tokens, ids out of range, or a mask that is not a left-aligned prefix of ones."""
        c = self.cfg
        ids = torch.as_tensor(input_ids).cpu()
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        if ids.dim() != 2 or ids.numel() == 0 or ids.is_floating_point():
            raise ValueError(f"input_ids must be a non-empty integer [B, T] tensor, got {tuple(ids.shape)} {ids.dtype}")
        ids = ids.long()
        B, T = ids.shape
        if T > c["max_position_embeddings"]:
            raise ValueError(f"{T} tokens exceed max_position_embeddings = {c['max_position_embeddings']}")
        if int(ids.min()) < 0 or int(ids.max()) >= c["vocab_size"]:
            raise ValueError(f"input ids outside [0, {c['vocab_size']})")
        if attention_mask is None:
            lens = torch.full((B,), T, dtype=torch.long)
        else:
            m = torch.as_tensor(attention_mask).cpu()
            if m.dim() == 1:
                m = m.unsqueeze(0)
            if tuple(m.shape) != (B, T):
                raise ValueError(f"attention_mask shape {tuple(m.shape)} != input_ids shape {(B, T)}")
            lens = m.long().sum(1)
            if not torch.equal(m.long(), (torch.arange(T)[None, :] < lens[:, None]).long()) or int(lens.min()) < 1:
                raise ValueError("attention_mask must be a left-aligned prefix of ones with at least one token per row")
        if token_type_ids is None:
            tt = torch.zeros_like(ids)
        else:
            tt = torch.as_tensor(token_type_ids).cpu().long().reshape(B, T)
            if int(tt.min()) < 0 or int(tt.max()) >= c["type_vocab_size"]:
                raise ValueError(f"token_type_ids outside [0, {c['type_vocab_size']})")
        return ids, tt, lens

    def _qkv(self, i):
        """Q, K and V of layer i as one Linear: the three weights concatenated and packed once per weights_key()."""
        key = ("qkv", i)
        if key not in self._active:
            p = f"encoder.layer.{i}.attention.self."
            w = torch.cat([self.P(p + n + ".weight").detach() for n in ("query", "key", "value")])
            b = torch.cat([self.P(p + n + ".bias").detach() for n in ("query", "key", "value")])
            self._active[key] = (ops.pack_weight(w, None, need_pb=False), b)
        return self._active[key]

    @torch.no_grad()
    def hidden_state(self, input_ids, attention_mask=None, token_type_ids=None, index=-3):
        """-> [B, T, H] fp32 on the model's device; each row equals transformers' `hidden_states[index]` of that row alone (rows
        past a row's length hold finite values that no valid row reads)."""
        c = self.cfg
        n = self.layers_for(index)
        ids, tt, lens = self.check_inputs(input_ids, attention_mask, token_type_ids)
        B, T = ids.shape
        dev = self.P("embeddings.word_embeddings.weight").device
        pos = torch.arange(T).expand(B, T)
        idx = torch.cat([ids.reshape(-1), tt.reshape(-1), pos.reshape(-1), lens]).to(dev)      # one H2D copy
        ids_d, tt_d, pos_d, lens_d = idx[:B * T].view(B, T), idx[B * T:2 * B * T].view(B, T), idx[2 * B * T:3 * B * T].view(B, T), idx[3 * B * T:]
        H, nh, eps = c["hidden_size"], c["num_attention_heads"], c["layer_norm_eps"]
        with self.inference_weights():
            # BertEmbeddings: (word + token type) + position, then LayerNorm
            x = ops.add(ops.embedding(self.P("embeddings.word_embeddings.weight"), ids_d),
                        ops.embedding(self.P("embeddings.token_type_embeddings.weight"), tt_d))
            h = ops.layernorm(x, self.P("embeddings.LayerNorm.weight"), self.P("embeddings.LayerNorm.bias"),
                              res=ops.embedding(self.P("embeddings.position_embeddings.weight"), pos_d), eps=eps)
            for i in range(n):
                p = f"encoder.layer.{i}."
                wqkv, bqkv = self._qkv(i)
                a = ops.attention_pad(ops.linear(h, wqkv, bqkv), heads=nh, lens=lens_d, scale=(H // nh) ** -0.5)
                a = ops.linear(a, self.w(p + "attention.output.dense", need_pb=False), self.b(p + "attention.output.dense"))
                h = ops.layernorm(h, self.P(p + "attention.output.LayerNorm.weight"), self.P(p + "attention.output.LayerNorm.bias"),
                                  res=a, eps=eps)
                f = ops.gelu(ops.linear(h, self.w(p + "intermediate.dense", need_pb=False), self.b(p + "intermediate.dense")))
                f = ops.linear(f, self.w(p + "output.dense", need_pb=False), self.b(p + "output.dense"))
                h = ops.layernorm(h, self.P(p + "output.LayerNorm.weight"), self.P(p + "output.LayerNorm.bias"), res=f, eps=eps)
            return h


# ---- phone-level expansion -------------------------------------------------------------------------------------------------
def phone_index(word2ph_list, T):
    """-> (idx int64 [B, P_max] of rows of the flattened [B * T] hidden states, [P_b]).  Phone k of row b that belongs to
    character i reads token i + 1 of row b; entries past P_b point at row b's token 0 and are zeroed after the gather."""
    P = [int(sum(w)) for w in word2ph_list]
    idx = torch.zeros((len(word2ph_list), max(P, default=0)), dtype=torch.long)
    for b, w in enumerate(word2ph_list):
        idx[b] = b * T
        idx[b, :P[b]] = b * T + 1 + torch.repeat_interleave(torch.arange(len(w)), torch.as_tensor(w, dtype=torch.long))
    return idx, P


def check_word2ph(text, word2ph, n_tokens, what="text"):
    """The reference's conditions: one word2ph entry per character of the text, and character i reads token i + 1, which must
    be a token of the sentence other than the final [SEP] (the reference raises IndexError there)."""
    if len(word2ph) != len(text):
        raise ValueError(f"{what}: text and word2ph not match ({len(text)} characters, {len(word2ph)} word2ph entries)")
    if len(word2ph) > n_tokens - 2:
        raise ValueError(f"{what}: character {n_tokens - 2} has no token ({n_tokens} tokens including [CLS] and [SEP])")
    if any(int(w) < 0 for w in word2ph):
        raise ValueError(f"{what}: negative word2ph entry")


@torch.no_grad()
def phone_features(hidden, word2ph_list):
    """hidden [B, T, H] (hidden_state output) -> ([B, H, P_max] channel-first, zero past P_b; [P_b]).  Pure copies: equal bit for
    bit to the reference's repeat of the same hidden state."""
    B, T, H = hidden.shape
    if len(word2ph_list) != B or any(len(w) > T - 2 for w in word2ph_list):
        raise ValueError(f"word2ph lists do not fit the {B} rows of {T} tokens")
    idx, P = phone_index(word2ph_list, T)
    if idx.shape[1] == 0:
        return hidden.new_zeros((B, H, 0)), P
    dev = hidden.device
    g = ops.embedding(hidden.reshape(B * T, H), idx.to(dev))
    g = ops.rowmask(g, torch.tensor(P, dtype=torch.int32).to(dev))
    return ops.to_channels_first(g), P


# ---- drop-ins ---------------------------------------------------------------------------------------------------------------
def _tokenize(text, tokenizer):
    enc = tokenizer(text, return_tensors="pt")
    return enc["input_ids"], enc.get("token_type_ids")


def get_bert_feature(text, word2ph, tokenizer, model):
    """`TextPreprocessor.get_bert_feature` / `Normalize._get_bert_feature`: -> [H, sum(word2ph)] fp32 on the model's device."""
    ids, tt = _tokenize(text, tokenizer)
    check_word2ph(text, word2ph, ids.shape[-1])
    f, P = phone_features(model.hidden_state(ids, token_type_ids=tt), [list(word2ph)])
    return f[0]


def get_bert_features(texts, word2phs, tokenizer, model, max_batch=32, max_tokens=8192):
    """get_bert_feature over many sentences -> list of [H, P_i] device tensors (views of the padded batch outputs).  One tokenizer
    call per text, as the reference makes; sentences are grouped longest first into right-padded batches of at most `max_batch`
    rows and `max_tokens` padded tokens, one forward each.  All inputs are checked before the first batch runs."""
    if len(texts) != len(word2phs):
        raise ValueError(f"{len(texts)} texts but {len(word2phs)} word2ph lists")
    enc = [_tokenize(t, tokenizer) for t in texts]
    for i, (t, w) in enumerate(zip(texts, word2phs)):
        check_word2ph(t, w, enc[i][0].shape[-1], what=f"text {i}")
        if enc[i][0].shape[-1] > model.cfg["max_position_embeddings"]:
            raise ValueError(f"text {i}: {enc[i][0].shape[-1]} tokens exceed max_position_embeddings = {model.cfg['max_position_embeddings']}")
    order = sorted(range(len(texts)), key=lambda i: -enc[i][0].shape[-1])
    out = [None] * len(texts)
    k = 0
    while k < len(order):
        Tm = enc[order[k]][0].shape[-1]
        grp = order[k:k + max(1, min(max_batch, max_tokens // Tm))]
        k += len(grp)
        ids = torch.zeros((len(grp), Tm), dtype=torch.long)
        tt = torch.zeros_like(ids)
        mask = torch.zeros_like(ids)
        for r, j in enumerate(grp):
            n = enc[j][0].shape[-1]
            ids[r, :n] = enc[j][0][0]
            if enc[j][1] is not None:
                tt[r, :n] = enc[j][1][0]
            mask[r, :n] = 1
        f, P = phone_features(model.hidden_state(ids, mask, tt), [list(word2phs[j]) for j in grp])
        for r, j in enumerate(grp):
            out[j] = f[r, :, :P[r]]
    return out


def write_bert_features(items, bert_dir, tokenizer, model, max_batch=32):
    """The BERT half of `Normalize._process_text` (normalize.py:108-130) for many utterances at once.  items: (name, norm_text,
    word2ph, n_phones, lang) tuples, `clean_text` already applied.  Only `zh` items whose `<bert_dir>/<name>.pt` does not exist
    are computed; each is saved as a contiguous CPU fp32 [H, P] tensor.  A word2ph that does not match its text, or a feature
    width that does not match n_phones, raises ValueError naming the utterance before anything runs.  -> names written."""
    todo = []
    for name, text, word2ph, n_phones, lang in items:
        name = os.path.basename(format_path(name))
        path = os.path.join(bert_dir, f"{name}.pt")
        if lang != "zh" or os.path.exists(path):
            continue
        if len(word2ph) != len(text):
            raise ValueError(f"{name}: text and word2ph not match")
        if sum(word2ph) != n_phones:
            raise ValueError(f"{name}: bert_feature and phones not match ({sum(word2ph)} != {n_phones})")
        todo.append((name, path, text, list(word2ph)))
    feats = get_bert_features([t[2] for t in todo], [t[3] for t in todo], tokenizer, model, max_batch=max_batch)
    for (name, path, _, _), f in zip(todo, feats):
        torch.save(f.cpu().contiguous(), path)
    return [t[0] for t in todo]
