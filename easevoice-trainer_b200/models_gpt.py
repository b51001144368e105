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
# infer_panel_batch_infer replays its step graph this many times between two reads of the finished flags: a read costs a host
# round trip (~tens of us), a step of 16 rows ~1 ms, so 8 replays keep the check under a few percent of the loop while a batch
# runs at most 7 steps past its last row's finish.
INFER_BATCH_K = 8
MAX_DECODE_STEPS = 1500                                            # t2s_model.py:646 (`for idx in range(1500)`)


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

    def _infer_layer(self, i, h, cache, n_prev, X=None, xl=None, yl=None, skip=None):
        """One post-LN block in inference.  Prompt pass (X given): h [B, L, D], prefix-LM attention, cache rows 0..L-1 filled
        (T2SBlock.process_prompt, t2s_model.py:121-185).  Token pass: h [B, 1, D], its in_proj row is appended to the cache
        and attends every cached position (decode_next_token, :187-221).  skip ([B, 2] int32, batched token pass): row b leaves
        out its text padding skip[b, 0] .. skip[b, 1] - 1, and the Linears run on ops.linear_rows (exact fp32 for up to 64 rows)."""
        p = f"h.layers.{i}."
        H = self.num_head
        lin = ops.linear if skip is None else ops.linear_rows
        qkv = lin(h, self.w(p + "self_attn.in_proj", suffix="_weight"), self.P(p + "self_attn.in_proj_bias"))
        L = qkv.shape[1]
        if torch.is_tensor(n_prev):                                # device-side position: the step is a replayed CUDA graph
            a = ops.attn_decode_dev(cache, n_prev, H, qkv, skip)
        elif X is not None:
            cache[:, n_prev:n_prev + L].copy_(qkv)
            a = ops.flash_attention(qkv, heads=H, prefix=X, xlen=xl, ylen=yl, p_drop=0.0, tag=f"gpt.infer{i}")
        else:
            cache[:, n_prev:n_prev + L].copy_(qkv)
            a = ops.attn_decode(cache, n_prev + 1, H)
        a = lin(a, self.w(p + "self_attn.out_proj"), self.b(p + "self_attn.out_proj"))
        h = ops.layernorm(h, self.P(p + "norm1.weight"), self.P(p + "norm1.bias"), res=a)
        f = lin(h, self.w(p + "linear1"), self.b(p + "linear1"), act=ops.ACT_RELU)
        f = lin(f, self.w(p + "linear2"), self.b(p + "linear2"))
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
        EOS is excluded for the first 11 steps (:835-836).
        Prompt-free decoding (prompts = None, TTS's ref_text_free mode; :796-803, :858-862): the prompt pass covers the text
        alone (full attention over it), the first logits come from the last text position, the token of step idx is embedded at
        pe[idx], and the result is (generated tokens without the last sample [1, n], 0); early_stop_num = 0 gives [1, 0].
        There is no CPU path: prompt-free inputs that are not CUDA tensors raise NotImplementedError."""
        if prompts is None and not (x.is_cuda and bert_feature.is_cuda):
            raise NotImplementedError("infer_panel: prompt-free decoding runs on CUDA tensors only (there is no CPU path)")
        assert x.shape[0] == 1 and (prompts is None or prompts.shape[0] == 1), "one utterance at a time, like infer_panel_naive"
        was_training = self.training
        self.eval()
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            dev = x.device
            D, V = self.model_dim, self.vocab_size
            X = x.shape[1]
            if prompts is None:                                          # :802: an empty token history
                y, Yp = torch.zeros((1, 0), device=dev, dtype=torch.int64), 0
            else:
                y, Yp = prompts.to(torch.int64), prompts.shape[1]
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
                # next input: embedding of the sampled token at position Yp + idx (t2s_model.py:858-859, x_scale = 1)
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
            return y[:, :-1], (0 if prompts is None else idx - 1)        # :861-863
        finally:
            self._active, self._memo_pack = None, False
            self.train(was_training)

    def infer_panel(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                    repetition_penalty=1.35, **kwargs):
        """t2s_model.py:869-882."""
        return self.infer_panel_naive(x, x_lens, prompts, bert_feature, top_k, top_p, early_stop_num, temperature,
                                      repetition_penalty, **kwargs)


    def infer_panel_naive_batched(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                                  repetition_penalty=1.35, **kwargs):
        """t2s_model.py:732-760: infer_panel_naive on each utterance in turn -> (list of 1-D y, list of idx).

        Prompt-free (prompts None, TTS's ref_text_free mode): x is a list of 1-D phoneme-id tensors or a padded [B, X] tensor,
        bert_feature a list of [1024, width of x[b]].  As in the reference, row b's text is all of x[b] (x[b].shape[0] positions):
        x_lens is not read, so the padding of a padded [B, X] tensor is decoded as text.  top_k must lie in [1, V].  On CUDA
        inputs every row is decoded together (_infer_ref_free_batched); each row gives what infer_panel_naive(prompts=None)
        gives on it alone, up to the sampling noise: (y_list, [0] * B), y_list[b] the generated tokens without the last sample.
        Other inputs keep the per-row loop, which has no CPU path and raises NotImplementedError."""
        if prompts is None:
            self._check_ref_free(x, bert_feature, top_k)
            if all(t.is_cuda for t in list(x) + list(bert_feature)):
                return self._infer_ref_free_batched(x, bert_feature, top_k, top_p, early_stop_num, temperature, repetition_penalty,
                                                    **kwargs)
        y_list, idx_list = [], []
        for i in range(len(x)):
            y, idx = self.infer_panel_naive(x[i].unsqueeze(0), x_lens[i], prompts[i].unsqueeze(0) if prompts is not None else None,
                                            bert_feature[i].unsqueeze(0), top_k, top_p, early_stop_num, temperature,
                                            repetition_penalty, **kwargs)
            y_list.append(y[0])
            idx_list.append(idx)
        return y_list, idx_list

    def _batch_state(self, dev, B, need_rows):
        """Per-layer caches [B, rows, 3 D] and the static buffers / graph of the batched token step, kept across calls while the
        parameters, B and the capacity allow (one state at a time: a new shape frees the previous one first)."""
        ver = sum(int(p._version) for p in self.parameters())
        st = self.__dict__.get("_batch_st")
        if st is not None and st["ver"] == ver and st["dev"] == dev and st["B"] == B and st["rows"] >= need_rows:
            return st
        self.__dict__.pop("_batch_st", None)
        rows = (need_rows + 63) // 64 * 64
        D, V, Vp = self.model_dim, self.vocab_size, (self.vocab_size + 3) // 4 * 4

        def z(*shape, dtype=torch.float32):
            return torch.zeros(shape, device=dev, dtype=dtype)
        st = dict(ver=ver, dev=dev, B=B, rows=rows, graphs={},
                  caches=[torch.empty((B, rows, 3 * D), device=dev, dtype=torch.float32) for _ in range(self.num_layers)],
                  n=z(1, dtype=torch.int32), x=z(B, 1, D), logits=z(B, Vp), skip=z(B, 2, dtype=torch.int32),
                  hist=z(B, rows, dtype=torch.int64), seen=z(B, (V + 31) // 32, dtype=torch.int32), fin=z(B, 2, dtype=torch.int32),
                  icfg=z(6, dtype=torch.int64), fcfg=z(3), pe=self.pe(rows, dev))
        self.__dict__["_batch_st"] = st
        return st

    def _batch_step_graph(self, st, head, eos_steps):
        """The step graph of `st` whose sampler excludes EOS at the steps idx < eos_steps (a kernel argument, fixed at capture:
        1 for infer_panel_batch_infer, 11 for prompt-free decoding), captured on first use."""
        if eos_steps not in st["graphs"]:
            st["graphs"][eos_steps] = self._capture_batch_step(st, head, eos_steps)
        return st["graphs"][eos_steps]

    def _capture_batch_step(self, st, head, eos_steps):
        """One decoding step of every row as one CUDA graph: sample from st["logits"] (writes the token, the finished flags and
        the next input row st["x"]), the 24 layers on st["x"], the vocabulary projection into st["logits"], position + 1."""
        emb = self.P("ar_audio_embedding.word_embeddings.weight")
        a_audio = self.P("ar_audio_position.alpha")

        def step():
            ops.sample_tokens(st["logits"], self.vocab_size, self.EOS, st["icfg"], st["fcfg"], st["n"], st["hist"], st["seen"],
                              st["fin"], emb, st["pe"], a_audio, st["x"], eos_steps=eos_steps)
            h = st["x"]
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, st["caches"][i], st["n"], skip=st["skip"])
            st["logits"].copy_(ops.linear_rows(h, head).view(st["logits"].shape))
            st["n"].add_(1)
        # warm-up and capture with every row marked finished (the sampler is then a no-op) at position 0 with nothing skipped;
        # the caller overwrites all of it before the first replay
        st["fin"].fill_(0)
        st["n"].zero_()
        st["skip"].zero_()
        side = torch.cuda.Stream(device=st["dev"])
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                              # outside capture: allocator, lazy inits, shared-memory opt-ins
            step()
        torch.cuda.current_stream().wait_stream(side)
        st["n"].zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        return g

    def _run_batch(self, st, graph, prefix, n0, top_k, early_stop_num, top_p, temperature, repetition_penalty, trace):
        """Decode every row of `st` (prompt pass done: caches, logits, n, skip, hist and seen set) until all have finished ->
        fin as a host list of [stop step, idx] per row.  The noise seed is drawn here, once per call, from torch's CUDA generator."""
        dev, K = st["dev"], INFER_BATCH_K
        st["fin"].fill_(-1)
        st["icfg"][0:1].copy_(torch.randint(0, 2 ** 62, (1,), device=dev, dtype=torch.int64))
        st["icfg"][1:].copy_(torch.tensor([prefix, n0, top_k, early_stop_num, MAX_DECODE_STEPS], dtype=torch.int64))
        st["fcfg"].copy_(torch.tensor([float(top_p), float(temperature), float(repetition_penalty)], dtype=torch.float32))
        while True:
            for _ in range(K if trace is None else 1):
                if trace is not None:
                    trace.append(st["logits"][:, :self.vocab_size].clone())
                graph.replay()
            if not bool((st["fin"][:, 0] < 0).any()):
                break
        return st["fin"].cpu().tolist()

    @torch.no_grad()
    def infer_panel_batch_infer(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                                repetition_penalty=1.35, **kwargs):
        """t2s_model.py:563-730: every sentence of a batch decoded together on one KV cache -> (y_list, idx_list), y_list[b] a
        1-D int64 device tensor (prompt + generated tokens), idx_list[b] an int.

        x: list of 1-D phoneme-id tensors, or a padded [B, X] tensor (row b then has width X); bert_feature: list of [1024, X_b]
        tensors of the same widths; x_lens [B]; prompts [B, Yp] (one prompt length for all rows, as TTS builds it with .expand);
        kwargs["max_len"] (default x_lens.max()) is the common text length the rows are right-padded to.  top_k must lie in
        [1, V].  With prompts None the call goes to infer_panel_naive_batched, as the reference does (:576-578; it does not
        pass repetition_penalty on, so the default 1.35 applies), which decodes the rows prompt-free.

        Restated from the reference, quirks included:
          - padded text positions (x_len_b <= t < max_len) are neither attended nor attending (:617-636); the position of row
            b's next input is pe[Yp + idx] for every row (:705);
          - EOS is excluded at step 0 only (`logits[:, :-1]` when idx == 0, :651-652; infer_panel_naive excludes it for the
            first 11 steps);
          - a row stops when its sampled token OR the argmax of its penalised logits is EOS (:662-672): the penalty is written
            into the logits in place (utils.py:123), so the argmax sees it;
          - a row finishing on EOS at step idx returns y[:-1] and idx - 1 (:673-677);
          - when early_stop_num is reached (idx + 1 > early_stop_num, :688) or at idx == 1499, every remaining row stops at that
            idx and returns y[:-1] and idx (:688-694);
          - decoding is capped at 1500 steps (:646); rows that never set their index would get 1499 (:708-712), which the cap
            already guarantees.
        Device path: one prompt pass over [B, max_len + Yp] on the training kernels (ragged prefix-LM flash attention with
        xlen = x_lens, ylen = Yp) fills per-layer caches of in_proj rows; then one CUDA graph per step (fused sampler + 24 layers
        of exact-fp32 row Linears and per-row-key decode attention + vocabulary projection) is replayed INFER_BATCH_K times
        between reads of the finished flags.  There is no per-token host sync.  Finished rows stay in the batch, frozen (the
        reference compacts them away; rows are independent, so the results are the same).  The caches hold
        max_len + Yp + min(1500, early_stop_num + 1) + INFER_BATCH_K rows (rounded up to 64) of 3 * 512 floats per layer and row:
        24 layers x B x rows x 6 KiB, e.g. 1.4 GiB for B = 16, max_len 120, Yp 150, early_stop_num 300 (640 rows).
        Random stream: the reference draws torch.exponential_ over a batch that shrinks as rows finish; here each Exp(1) draw is
        a counter-based function of (seed, row, step, token id) with the seed drawn once per call from torch's CUDA default
        generator, so torch.manual_seed still makes a run reproducible but sampled tokens differ from the reference's.
        Greedy decoding (top_k = 1) does not depend on the stream.  kwargs["trace"] (a list, tests) receives the raw [B, V]
        logits of every step and makes the host check the flags after every step."""
        if prompts is None:
            return self.infer_panel_naive_batched(x, x_lens, prompts, bert_feature, top_k=top_k, top_p=top_p,
                                                  early_stop_num=early_stop_num, temperature=temperature, **kwargs)
        B = len(x)
        V, EOS, D = self.vocab_size, self.EOS, self.model_dim
        if int(top_k) != top_k or not 1 <= top_k <= V:
            raise ValueError(f"infer_panel_batch_infer: top_k must be an integer in [1, {V}], got {top_k!r}")
        top_k = int(top_k)
        if len(bert_feature) != B or prompts.dim() != 2 or prompts.shape[0] != B or len(x_lens) != B:
            raise ValueError("infer_panel_batch_infer: x, x_lens, prompts and bert_feature must have one entry per row")
        if B > 64:                                                 # the row Linears take 64 rows per launch
            out = [self.infer_panel_batch_infer(x[i:i + 64], x_lens[i:i + 64], prompts[i:i + 64], bert_feature[i:i + 64], top_k,
                                                top_p, early_stop_num, temperature, repetition_penalty,
                                                **dict(kwargs, max_len=kwargs.get("max_len", max(int(v) for v in x_lens))))
                   for i in range(0, B, 64)]
            return [y for o in out for y in o[0]], [i for o in out for i in o[1]]
        dev = prompts.device
        xl_host = [int(v) for v in x_lens]
        max_len = int(kwargs.get("max_len", max(xl_host)))
        rows = [x[b] for b in range(B)]
        for b in range(B):
            if rows[b].dim() != 1 or bert_feature[b].shape != (1024, rows[b].shape[0]) or not 1 <= xl_host[b] <= rows[b].shape[0] <= max_len:
                raise ValueError(f"infer_panel_batch_infer: row {b}: x {tuple(rows[b].shape)}, bert_feature {tuple(bert_feature[b].shape)}, "
                                 f"x_len {xl_host[b]}, max_len {max_len}")
        Yp = prompts.shape[1]
        L0 = max_len + Yp
        cap = MAX_DECODE_STEPS if early_stop_num == -1 else min(MAX_DECODE_STEPS, early_stop_num + 1)
        K = INFER_BATCH_K
        was_training = self.training
        self.eval()
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            xp = torch.zeros((B, max_len), device=dev, dtype=torch.int64)
            bp = torch.zeros((B, 1024, max_len), device=dev, dtype=torch.float32)
            for b in range(B):
                xp[b, :rows[b].shape[0]] = rows[b]
                bp[b, :, :rows[b].shape[0]] = bert_feature[b]
            st = self._batch_state(dev, B, L0 + cap + K)
            Vp = st["logits"].shape[1]
            head = self.w("ar_predict_layer", pad0=Vp)
            graph = self._batch_step_graph(st, head, 1)
            # prompt pass (process_prompt with the padded mask, :596-646)
            y = prompts.to(torch.int64)
            xe = self._embed_text(xp, bp, False)
            ye = ops.embedding(self.P("ar_audio_embedding.word_embeddings.weight"), y)
            h = ops.gpt_embed(xe, ye, self.P("ar_text_position.alpha"), self.P("ar_audio_position.alpha"), st["pe"])
            xl = torch.tensor(xl_host, device=dev, dtype=torch.int64)
            yl = torch.full((B,), Yp, device=dev, dtype=torch.int64)
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, st["caches"][i], 0, max_len, xl, yl)
            st["logits"].copy_(ops.linear_rows(h[:, -1:].contiguous(), head).view(B, Vp))
            # per-call state of the step graph
            st["n"].fill_(L0)
            st["skip"].copy_(torch.tensor([[v, max_len] for v in xl_host], dtype=torch.int32))
            st["hist"][:, :Yp].copy_(y)
            bits = torch.zeros((B, st["seen"].shape[1] * 32), device=dev, dtype=torch.int64).scatter_(1, y, 1)
            words = (bits.view(B, -1, 32) << torch.arange(32, device=dev, dtype=torch.int64)).sum(-1)
            st["seen"].copy_(torch.where(words >= 2 ** 31, words - 2 ** 32, words))      # uint32 bit patterns as int32
            fin = self._run_batch(st, graph, Yp, L0, top_k, early_stop_num, top_p, temperature, repetition_penalty, kwargs.get("trace"))
            return [st["hist"][b, :Yp + fin[b][0]].clone() for b in range(B)], [f[1] for f in fin]
        finally:
            self._active, self._memo_pack = None, False
            self.train(was_training)

    def _check_ref_free(self, x, bert_feature, top_k):
        """Argument checks of prompt-free batched decoding (ValueError, before anything runs)."""
        V = self.vocab_size
        if int(top_k) != top_k or not 1 <= top_k <= V:
            raise ValueError(f"infer_panel_naive_batched: top_k must be an integer in [1, {V}], got {top_k!r}")
        if len(bert_feature) != len(x):
            raise ValueError("infer_panel_naive_batched: x and bert_feature must have one entry per row")
        for b in range(len(x)):
            if x[b].dim() != 1 or x[b].shape[0] < 1 or tuple(bert_feature[b].shape) != (1024, x[b].shape[0]):
                raise ValueError(f"infer_panel_naive_batched: row {b}: x {tuple(x[b].shape)}, bert_feature {tuple(bert_feature[b].shape)}")

    @torch.no_grad()
    def _infer_ref_free_batched(self, x, bert_feature, top_k, top_p, early_stop_num, temperature, repetition_penalty, **kwargs):
        """infer_panel_naive_batched with prompts None on CUDA inputs: infer_panel_naive(prompts=None) (t2s_model.py:762-863) for
        every row at once, on the machinery of infer_panel_batch_infer.  Row b has len_b = x[b].shape[0] text positions.
          - Prompt pass: one pass over the right-padded [B, max_len] text (prefix-LM flash attention with X = max_len,
            xlen = len_b, ylen = 0: each row attends its own text, bidirectionally); row b's first logits come from its last
            text position h[b, len_b - 1].  max_len = max(kwargs["max_len"], longest row); it does not change the results.
          - Step idx: the token goes to cache row max_len + idx and is embedded at pe[idx] (y_len = 0, :858-859); each row leaves
            out its text padding len_b .. max_len - 1; EOS is excluded for idx < 11 (:835-836); a row stops when its sample or
            the argmax of its penalised logits is EOS, or at idx + 1 > early_stop_num, or at idx 1499.
          - -> (y_list, [0] * B): y_list[b] the row's generated tokens without the last sample (:861-862).
        Noise: counter-based Exp(1) draws as in infer_panel_batch_infer, seeded once per call from torch's CUDA generator, so
        torch.manual_seed reproduces a run and greedy decoding does not depend on it.  kwargs["trace"] as there.  Batches of more
        than 64 rows run in chunks of 64."""
        B = len(x)
        max_len = max([int(kwargs.get("max_len", 0))] + [int(x[b].shape[0]) for b in range(B)])
        if B > 64:                                                 # the row Linears take 64 rows per launch
            out = [self._infer_ref_free_batched(x[i:i + 64], bert_feature[i:i + 64], top_k, top_p, early_stop_num, temperature,
                                                repetition_penalty, **dict(kwargs, max_len=max_len))
                   for i in range(0, B, 64)]
            return [y for o in out for y in o[0]], [i for o in out for i in o[1]]
        dev = x[0].device
        lens = [int(x[b].shape[0]) for b in range(B)]
        cap = MAX_DECODE_STEPS if early_stop_num == -1 else min(MAX_DECODE_STEPS, early_stop_num + 1)
        was_training = self.training
        self.eval()
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            xp = torch.zeros((B, max_len), device=dev, dtype=torch.int64)
            bp = torch.zeros((B, 1024, max_len), device=dev, dtype=torch.float32)
            for b in range(B):
                xp[b, :lens[b]] = x[b]
                bp[b, :, :lens[b]] = bert_feature[b]
            st = self._batch_state(dev, B, max_len + cap + INFER_BATCH_K)
            Vp = st["logits"].shape[1]
            head = self.w("ar_predict_layer", pad0=Vp)
            graph = self._batch_step_graph(st, head, 11)
            # prompt pass over the text alone (:796-803, :825)
            xe = self._embed_text(xp, bp, False)
            ye = ops.embedding(self.P("ar_audio_embedding.word_embeddings.weight"), torch.zeros((B, 0), device=dev, dtype=torch.int64))
            h = ops.gpt_embed(xe, ye, self.P("ar_text_position.alpha"), self.P("ar_audio_position.alpha"), st["pe"])
            xl = torch.tensor(lens, device=dev, dtype=torch.int64)
            yl = torch.zeros((B,), device=dev, dtype=torch.int64)
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, st["caches"][i], 0, max_len, xl, yl)
            last = ops.slice_rows(h, xl - 1, 1)                    # [B, 1, D]: each row's last text position
            st["logits"].copy_(ops.linear_rows(last, head).view(B, Vp))
            # per-call state of the step graph: no history, position max_len, text padding skipped
            st["n"].fill_(max_len)
            st["skip"].copy_(torch.tensor([[v, max_len] for v in lens], dtype=torch.int32))
            st["seen"].zero_()
            fin = self._run_batch(st, graph, 0, max_len, int(top_k), early_stop_num, top_p, temperature, repetition_penalty,
                                  kwargs.get("trace"))
            return [st["hist"][b, :fin[b][0]].clone() for b in range(B)], [0] * B
        finally:
            self._active, self._memo_pack = None, False
            self.train(was_training)


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
