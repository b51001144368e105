"""Stage-1 AR semantic-token GPT on the sm_90a kernels.

Mirror of /root/reference/src/easevoice/soundstorm/auto_reg/models/t2s_model.py `Text2SemanticDecoder` (training
path: forward_old :431-490) with the reference's parameter names, shapes and dtypes, so `state_dict()` is
interchangeable (Lightning checkpoints carry these keys under a "model." prefix, t2s_lightning_module.py:26).

Execution is channels-last [B, L, D] fp32 throughout:
  bert_proj / in_proj / out_proj / linear1(+ReLU) / linear2 / ar_predict_layer  -> ops.linear (wgmma TF32 GEMM tiles)
  prefix-LM masked SDPA with probability dropout                               -> ops.flash_attention (fused, O(L) memory)
  residual + post-LayerNorm (transformer.py:300-315, norm_first=False)          -> ops.layernorm(res=...)
  token embeddings, alpha * sinusoid + concat                                   -> ops.embedding / ops.gpt_embed
  CrossEntropyLoss(sum) + top-3 accuracy ignoring EOS                           -> ops.ce_sum_topk
The reference hard-codes dropout 0.1 in the positional embeddings, attention probabilities and the three layer
dropouts even though configs/gpt.yaml says `dropout: 0` (t2s_model.py:276-293); `layer_dropout` reproduces that
(default 0.1) and can be set to 0 for parity runs.
"""
import math
import os

import torch

from . import ops
from .models import ParamTree


INFER_GRAPH = os.environ.get("EVK_INFER_GRAPH", "1") != "0"      # token step of infer_panel as one replayed CUDA graph


def sine_table(length, dim):
    """embedding.py:53-69 computed the same way (fp32 torch ops on the host), uploaded once as a constant."""
    pos = torch.arange(0, length, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe = torch.zeros(length, dim)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


class Text2SemanticDecoder(ParamTree):
    """t2s_model.py:255-300 (constructor contract: config["model"] keys)."""

    def __init__(self, config, norm_first=False, top_k=3, layer_dropout=0.1, seed=None):
        super().__init__()
        m = config["model"]
        assert not norm_first, "the reference trains the post-LN variant only"
        self.model_dim, self.embedding_dim = m["hidden_dim"], m["embedding_dim"]
        self.num_head, self.num_layers = m["head"], m["n_layer"]
        self.vocab_size, self.phoneme_vocab_size = m["vocab_size"], m["phoneme_vocab_size"]
        self.p_dropout, self.EOS, self.top_k = float(m["dropout"]), m["EOS"], top_k
        self.layer_dropout = float(layer_dropout)
        assert self.EOS == self.vocab_size - 1
        assert self.model_dim == self.embedding_dim and self.model_dim // self.num_head == 32, "head dim 32 kernels"
        D, F = self.model_dim, self.model_dim * 4
        gen = torch.Generator().manual_seed(0 if seed is None else seed)

        def uni(shape, bound):
            return (torch.rand(shape, generator=gen) * 2 - 1) * bound

        def xavier(shape):
            return uni(shape, math.sqrt(6.0 / (shape[0] + shape[1])))

        self._register("bert_proj.weight", uni((D, 1024), 1 / math.sqrt(1024)))
        self._register("bert_proj.bias", uni((D,), 1 / math.sqrt(1024)))
        self._register("ar_text_embedding.word_embeddings.weight", torch.randn((self.phoneme_vocab_size, D), generator=gen))
        self._register("ar_text_position.alpha", torch.ones(1))
        self._register("ar_audio_embedding.word_embeddings.weight", torch.randn((self.vocab_size, D), generator=gen))
        self._register("ar_audio_position.alpha", torch.ones(1))
        for i in range(self.num_layers):
            p = f"h.layers.{i}."
            self._register(p + "self_attn.in_proj_weight", xavier((3 * D, D)))
            self._register(p + "self_attn.in_proj_bias", torch.zeros(3 * D))
            self._register(p + "self_attn.out_proj.weight", uni((D, D), 1 / math.sqrt(D)))
            self._register(p + "self_attn.out_proj.bias", torch.zeros(D))
            self._register(p + "linear1.weight", uni((F, D), 1 / math.sqrt(D)))
            self._register(p + "linear1.bias", uni((F,), 1 / math.sqrt(D)))
            self._register(p + "linear2.weight", uni((D, F), 1 / math.sqrt(F)))
            self._register(p + "linear2.bias", uni((D,), 1 / math.sqrt(F)))
            self._register(p + "norm1.weight", torch.ones(D))
            self._register(p + "norm1.bias", torch.zeros(D))
            self._register(p + "norm2.weight", torch.ones(D))
            self._register(p + "norm2.bias", torch.zeros(D))
        self._register("ar_predict_layer.weight", uni((self.vocab_size, D), 1 / math.sqrt(D)))
        self._pe = None

    def pe(self, length, device):
        if self._pe is None or self._pe.shape[0] < length or self._pe.device != device:
            self._pe = sine_table(max(length, 2048), self.model_dim).to(device)
        return self._pe

    def _drop(self, x, tag):
        return ops.dropout(x, self.layer_dropout, tag) if (self.training and self.layer_dropout > 0) else x

    def make_targets(self, y, y_lens):
        """pad_y_eos (t2s_model.py:557-561) on the host-visible int tensors (exact integer work, tiny)."""
        Y = y.shape[1]
        ymask = (torch.arange(Y, device=y.device)[None, :] >= y_lens[:, None]).to(torch.int64)
        codes = y.to(torch.int64) * (1 - ymask)
        tg = torch.nn.functional.pad(codes, (0, 1), value=0) + self.EOS * torch.nn.functional.pad(ymask, (0, 1), value=1)
        return tg[:, :-1].contiguous(), tg[:, 1:].contiguous()

    def _decode(self, xe, y_in, x_lens, y_lens, X, tagp=""):
        """embedded text prefix + shifted semantic tokens -> padded logits [B, Y, Vp] (t2s_model.py:462-487)."""
        B, Y = y_in.shape
        D, H, dev = self.model_dim, self.num_head, xe.device
        ye = ops.embedding(self.P("ar_audio_embedding.word_embeddings.weight"), y_in)
        h = ops.gpt_embed(xe, ye, self.P("ar_text_position.alpha"), self.P("ar_audio_position.alpha"), self.pe(max(X, Y), dev))
        h = self._drop(h, tagp + "gpt.pos")
        p_attn = self.layer_dropout if self.training else 0.0
        for i in range(self.num_layers):
            p = f"h.layers.{i}."
            qkv = ops.linear(h, self.w(p + "self_attn.in_proj", suffix="_weight"), self.P(p + "self_attn.in_proj_bias"))
            a = ops.flash_attention(qkv, heads=H, prefix=X, xlen=x_lens, ylen=y_lens, p_drop=p_attn, tag=f"{tagp}gpt.attn{i}")
            a = ops.linear(a, self.w(p + "self_attn.out_proj"), self.b(p + "self_attn.out_proj"))
            pd = self.layer_dropout if self.training else 0.0
            # the three layer dropouts are fused: into the two LayerNorm kernels (residual branch) and into linear1's epilogue
            h = ops.layernorm(h, self.P(p + "norm1.weight"), self.P(p + "norm1.bias"), res=a, res_drop=(pd, f"{tagp}gpt.d1.{i}"))
            f = ops.linear(h, self.w(p + "linear1"), self.b(p + "linear1"), act=ops.ACT_RELU, drop=(pd, f"{tagp}gpt.df.{i}"))
            f = ops.linear(f, self.w(p + "linear2"), self.b(p + "linear2"))
            h = ops.layernorm(h, self.P(p + "norm2.weight"), self.P(p + "norm2.bias"), res=f, res_drop=(pd, f"{tagp}gpt.d2.{i}"))
        key = (B, X, str(dev))
        if getattr(self, "_xoff_key", None) != key:
            self._xoff, self._xoff_key = torch.full((B,), X, device=dev, dtype=torch.int64), key
        hy = ops.slice_rows(h, self._xoff, Y)
        Vp = (self.vocab_size + 3) // 4 * 4
        return ops.linear(hy, self.w("ar_predict_layer", pad0=Vp))

    def _embed_text(self, x, bert_feature, bert_channels_last):
        bert_cl = bert_feature if bert_channels_last else ops.to_channels_last(bert_feature)
        xe = ops.embedding(self.P("ar_text_embedding.word_embeddings.weight"), x.to(torch.int64))
        return ops.linear(bert_cl, self.w("bert_proj", need_pb=False), self.b("bert_proj"), res=xe)

    def forward(self, x, x_lens, y, y_lens, bert_feature, reject=None, bert_channels_last=False):
        """DPO variant (t2s_model.py:393-429): CE(sum) on the given y plus a reference-free DPO term (beta 0.2) against
        a synthetically corrupted `reject` = (reject_y, reject_y_lens); built by `make_reject_y` when not given.
        -> (loss, acc)."""
        if reject is None:
            reject = make_reject_y(y, y_lens)
        ry, ryl = reject
        B, X = x.shape
        x_lens, y_lens, ryl = [t.to(torch.int64).contiguous() for t in (x_lens, y_lens, ryl)]
        y_in, tg = self.make_targets(y, y_lens)
        ry_in, rtg = self.make_targets(ry, ryl)
        self.begin_pack()
        try:
            return self._forward_dpo(x, bert_feature, bert_channels_last, y_in, tg, ry_in, rtg, x_lens, y_lens, ryl, X)
        finally:
            self.end_pack()

    def _forward_dpo(self, x, bert_feature, bert_channels_last, y_in, tg, ry_in, rtg, x_lens, y_lens, ryl, X):
        # the text prefix is embedded once per branch in the reference (two make_input_data calls); the branches only share
        # weights, so the second pass re-runs it to keep the dropout streams independent as well
        lc = self._decode(self._embed_text(x, bert_feature, bert_channels_last), y_in, x_lens, y_lens, X)
        lr_ = self._decode(self._embed_text(x, bert_feature, bert_channels_last), ry_in, x_lens, ryl, X, tagp="rej.")
        loss, metrics = ops.dpo_ce(lc, tg, lr_, rtg, self.top_k, self.EOS, V=self.vocab_size, beta=0.2)
        self.last_logits, self.last_dpo = lc.detach(), metrics
        return loss, metrics[2]

    def forward_old(self, x, x_lens, y, y_lens, bert_feature, targets=None, bert_channels_last=False):
        """-> (loss, acc) like t2s_model.py:431-490; `loss` is differentiable, `acc` a device scalar.
        bert_feature: [B, 1024, X] (reference layout), or [B, X, 1024] with bert_channels_last=True."""
        B, X = x.shape
        x_lens, y_lens = x_lens.to(torch.int64).contiguous(), y_lens.to(torch.int64).contiguous()
        y_in, tg = self.make_targets(y, y_lens) if targets is None else targets
        self.begin_pack()                      # all 147 weight packs of the step in one launch (ops.PackPlan)
        try:
            logits = self._decode(self._embed_text(x, bert_feature, bert_channels_last), y_in, x_lens, y_lens, X)
        finally:
            self.end_pack()
        loss, out2 = ops.ce_sum_topk(logits, tg.reshape(-1), self.top_k, self.EOS, V=self.vocab_size)
        self.last_logits = logits.detach()        # detached: a retained graph would pin AccumulateGrad nodes to this stream
        return loss, out2[1]


    # ---- inference: KV-cache decoding (SURVEY 8 row f4) -------------------------------------------------------------------
    @staticmethod
    def logits_to_probs(logits, previous_tokens=None, temperature=1.0, top_k=None, top_p=None, repetition_penalty=1.0):
        """utils.py:109-145 on a [1, V] row of logits (torch ops on the device: a 1 025-element row per token is not a kernel
        problem).  Same order of operations: repetition penalty, nucleus cut, temperature, top-k cut, softmax."""
        if previous_tokens is not None and repetition_penalty != 1.0:
            previous_tokens = previous_tokens.long()
            score = torch.gather(logits, dim=1, index=previous_tokens)
            score = torch.where(score < 0, score * repetition_penalty, score / repetition_penalty)
            logits.scatter_(dim=1, index=previous_tokens, src=score)   # IN PLACE, like the reference: the caller's EOS test (argmax of
            #                                                            the same tensor) therefore sees the penalised logits
        if top_p is not None and top_p < 1.0:
            sorted_logits, sorted_indices = torch.sort(logits, descending=True)
            cum = torch.cumsum(torch.softmax(sorted_logits, dim=-1), dim=-1)
            remove = cum > top_p
            remove[:, 0] = False
            logits = logits.masked_fill(remove.scatter(dim=1, index=sorted_indices, src=remove), -float("inf"))
        logits = logits / max(temperature, 1e-5)
        if top_k is not None:
            v, _ = torch.topk(logits, min(top_k, logits.size(-1)))
            logits = torch.where(logits < v[:, -1].unsqueeze(-1), -float("inf"), logits)
        return torch.softmax(logits, dim=-1)

    def _infer_layer(self, i, h, cache, n_prev, X=None, xl=None, yl=None):
        """One post-LN block in inference.  Prompt pass (X given): h [1, L, D], prefix-LM attention, cache rows 0..L-1 filled
        (T2SBlock.process_prompt, t2s_model.py:121-185).  Token pass: h [1, 1, D], its in_proj row is appended to the cache
        and attends every cached position (decode_next_token, :187-221)."""
        p = f"h.layers.{i}."
        H = self.num_head
        qkv = ops.linear(h, self.w(p + "self_attn.in_proj", suffix="_weight"), self.P(p + "self_attn.in_proj_bias"))
        L = qkv.shape[1]
        if torch.is_tensor(n_prev):                                # device-side position: the step is a replayed CUDA graph
            a = ops.attn_decode_dev(cache, n_prev, H, qkv)
        elif X is not None:
            cache[:, n_prev:n_prev + L].copy_(qkv)
            a = ops.flash_attention(qkv, heads=H, prefix=X, xlen=xl, ylen=yl, p_drop=0.0, tag=f"gpt.infer{i}")
        else:
            cache[:, n_prev:n_prev + L].copy_(qkv)
            a = ops.attn_decode(cache, n_prev + 1, H)
        a = ops.linear(a, self.w(p + "self_attn.out_proj"), self.b(p + "self_attn.out_proj"))
        h = ops.layernorm(h, self.P(p + "norm1.weight"), self.P(p + "norm1.bias"), res=a)
        f = ops.linear(h, self.w(p + "linear1"), self.b(p + "linear1"), act=ops.ACT_RELU)
        f = ops.linear(f, self.w(p + "linear2"), self.b(p + "linear2"))
        return ops.layernorm(h, self.P(p + "norm2.weight"), self.P(p + "norm2.bias"), res=f)

    def _infer_state(self, dev, need_rows):
        """Per-layer caches of in_proj rows + the static buffers / graph of the token step, kept across calls while the
        parameters (version counters) and the capacity allow."""
        ver = sum(int(p._version) for p in self.parameters())
        st = self.__dict__.get("_infer_st")
        if st is None or st["ver"] != ver or st["dev"] != dev or st["rows"] < need_rows:
            rows = (need_rows + 511) // 512 * 512
            D, Vp = self.model_dim, (self.vocab_size + 3) // 4 * 4
            st = dict(ver=ver, dev=dev, rows=rows, graph=None,
                      caches=[torch.empty((1, rows, 3 * D), device=dev, dtype=torch.float32) for _ in range(self.num_layers)],
                      n=torch.zeros(1, device=dev, dtype=torch.int32), x=torch.zeros((1, 1, D), device=dev, dtype=torch.float32),
                      logits=torch.zeros((1, 1, Vp), device=dev, dtype=torch.float32))
            self.__dict__["_infer_st"] = st
        return st

    def _capture_token_step(self, st, head):
        def step():
            h = st["x"]
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, st["caches"][i], st["n"])
            st["logits"].copy_(ops.linear(h, head))
            st["n"].add_(1)
        n0 = st["n"].clone()
        side = torch.cuda.Stream(device=st["dev"])
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                              # warm-up outside capture (allocator, lazy inits)
            step()
        torch.cuda.current_stream().wait_stream(side)
        st["n"].copy_(n0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        st["n"].copy_(n0)                                          # capture does not execute: the position is still n0
        st["graph"] = g

    @torch.no_grad()
    def infer_panel_naive(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                          repetition_penalty=1.35, max_steps=1500, trace=None, **kwargs):
        """t2s_model.py:762-867: one utterance (x [1, X] phoneme ids, bert_feature [1, 1024, X], prompts [1, Yp] semantic
        tokens of the reference audio) -> (y[:, :-1] = prompt + generated tokens, index of the last generated token).
        The prompt pass runs the training forward's kernels and fills a per-layer cache of in_proj rows; every further token is
        24 x (6 Linear launches on a one-row operand + one KV-cache attention + two LayerNorms).  Sampling follows utils.py:102-157
        (exponential-race multinomial on the device).  `trace` (list) receives the [1, V] logits of every step (tests).
        Prompt-free decoding (prompts = None) is not implemented on this path."""
        if prompts is None:
            raise NotImplementedError("infer_panel: prompt-free decoding is not implemented on the sm_90a path")
        assert x.shape[0] == 1 and prompts.shape[0] == 1, "one utterance at a time, like infer_panel_naive"
        was_training = self.training
        self.eval()
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            dev = x.device
            D, V = self.model_dim, self.vocab_size
            X, Yp = x.shape[1], prompts.shape[1]
            y = prompts.to(torch.int64)
            xe = self._embed_text(x, bert_feature, False)
            ye = ops.embedding(self.P("ar_audio_embedding.word_embeddings.weight"), y)
            pe = self.pe(max(X, Yp + max_steps + 2), dev)
            h = ops.gpt_embed(xe, ye, self.P("ar_text_position.alpha"), self.P("ar_audio_position.alpha"), pe)
            L0 = X + Yp
            st = self._infer_state(dev, L0 + max_steps + 1)
            caches = st["caches"]
            xl = torch.full((1,), X, device=dev, dtype=torch.int64)
            yl = torch.full((1,), Yp, device=dev, dtype=torch.int64)
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, caches[i], 0, X, xl, yl)
            n = L0
            Vp = (V + 3) // 4 * 4
            head = self.w("ar_predict_layer", pad0=Vp)
            emb = self.P("ar_audio_embedding.word_embeddings.weight")
            a_audio = self.P("ar_audio_position.alpha")
            prefix_len = Yp
            stop = False
            idx = 0
            use_graph = INFER_GRAPH
            if use_graph:
                st["n"].fill_(n)
                st["logits"].copy_(ops.linear(h[:, -1:].contiguous(), head))
            else:
                last = h[:, -1:].contiguous()
            for idx in range(max_steps):
                logits = (st["logits"].clone() if use_graph else ops.linear(last, head))[:, 0, :V]      # [1, V]
                if trace is not None:
                    trace.append(logits.clone())
                if idx < 11:                                                     # at least 10 tokens before EOS may win (:835-836)
                    logits = logits[:, :-1]
                probs = self.logits_to_probs(logits, y, temperature=temperature, top_k=top_k, top_p=top_p,
                                             repetition_penalty=repetition_penalty)
                q = torch.empty_like(probs).exponential_(1)
                samples = torch.argmax(probs / q, dim=-1, keepdim=True).to(torch.int64)
                y = torch.cat([y, samples], dim=1)
                if early_stop_num != -1 and (y.shape[1] - prefix_len) > early_stop_num:
                    stop = True
                if int(torch.argmax(logits, dim=-1)[0]) == self.EOS or int(samples[0, 0]) == self.EOS:
                    stop = True
                if stop:
                    break
                # next input: embedding of the sampled token at position Yp + idx (t2s_model.py:861-862, x_scale = 1)
                last = (emb[y[:, -1:]] + a_audio * pe[Yp + idx]).contiguous()
                if use_graph:
                    # the whole 24-layer token step (+ the vocabulary projection) is ONE graph replay; the position lives in
                    # device memory (st["n"], advanced inside the graph), the token embedding is the only input
                    st["x"].copy_(last)
                    if st["graph"] is None:
                        self._capture_token_step(st, head)
                    st["graph"].replay()
                else:
                    for i in range(self.num_layers):
                        last = self._infer_layer(i, last, caches[i], n)
                    n += 1
            return y[:, :-1], idx - 1
        finally:
            self._active, self._memo_pack = None, False
            self.train(was_training)

    def infer_panel(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                    repetition_penalty=1.35, **kwargs):
        """t2s_model.py:869-882."""
        return self.infer_panel_naive(x, x_lens, prompts, bert_feature, top_k, top_p, early_stop_num, temperature,
                                      repetition_penalty, **kwargs)


def make_reject_y(y_o, y_lens, generator=None):
    """utils.py:195-232: per item, duplicate a random span of the PADDED row (the reference's `randint(0, 1)` always picks
    the repeat branch); rows are re-padded with 0 to the longest result.  Host-side integer work, as in the reference."""
    rows, lens = [], []
    for b in range(len(y_lens)):
        y = y_o[b]
        i0, i1 = sorted(torch.randint(0, len(y), size=(2,), generator=generator).tolist())
        rows.append(torch.cat([y[:i0], y[i0:i1], y[i0:i1], y[i1:]]))
        lens.append(len(rows[-1]))
    Ym = max(lens)
    out = torch.zeros((len(rows), Ym), dtype=y_o.dtype, device=y_o.device)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out, torch.tensor(lens, device=y_lens.device)
