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

import torch

from . import ops
from .models import ParamTree


# batched decoding replays its step graph this many times between two reads of the finished flags: a read costs a host
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
    def _infer_layer(self, i, h, cache, n_dev, skip=None, X=None, xl=None, yl=None):
        """One post-LN block in inference.  Prompt pass (n_dev None): h [B, L, D], prefix-LM attention over X text positions
        (per-row lengths xl / yl), cache rows 0..L-1 filled (T2SBlock.process_prompt, t2s_model.py:121-185).  Token step (n_dev an
        int32 device scalar, so the step can be a replayed CUDA graph): h [B, 1, D], its in_proj row is appended to the cache at
        *n_dev and attends every cached position (decode_next_token, :187-221); row b leaves out its text padding
        skip[b, 0] .. skip[b, 1] - 1, and the Linears run on ops.linear_rows (exact fp32 for up to 64 rows)."""
        p = f"h.layers.{i}."
        H = self.num_head
        lin = ops.linear if n_dev is None else ops.linear_rows
        qkv = lin(h, self.w(p + "self_attn.in_proj", suffix="_weight"), self.P(p + "self_attn.in_proj_bias"))
        if n_dev is None:
            cache[:, :qkv.shape[1]].copy_(qkv)
            a = ops.flash_attention(qkv, heads=H, prefix=X, xlen=xl, ylen=yl, p_drop=0.0, tag=f"gpt.infer{i}")
        else:
            a = ops.attn_decode_dev(cache, n_dev, H, qkv, skip)
        a = lin(a, self.w(p + "self_attn.out_proj"), self.b(p + "self_attn.out_proj"))
        h = ops.layernorm(h, self.P(p + "norm1.weight"), self.P(p + "norm1.bias"), res=a)
        f = lin(h, self.w(p + "linear1"), self.b(p + "linear1"), act=ops.ACT_RELU)
        f = lin(f, self.w(p + "linear2"), self.b(p + "linear2"))
        return ops.layernorm(h, self.P(p + "norm2.weight"), self.P(p + "norm2.bias"), res=f)

    @torch.no_grad()
    def infer_panel_naive(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                          repetition_penalty=1.35, max_steps=1500, trace=None, **kwargs):
        """t2s_model.py:762-867: one utterance (x [1, X] phoneme ids, bert_feature [1, 1024, X], prompts [1, Yp] semantic
        tokens of the reference audio) -> (y[:, :-1] = prompt + generated tokens, index of the last generated token).
        A batch of one on the batched decoder (_decode_batch): the prompt pass runs the training forward's kernels and fills a
        per-layer cache of in_proj rows; every further token is one replayed CUDA graph (fused sampler, 24 layers of one-row
        Linears and KV-cache attention, vocabulary projection).  EOS is excluded for the first 11 steps (:835-836); a finish at
        step idx, on EOS or at early_stop_num / max_steps, returns idx - 1 (:861-863).  top_k: an integer >= 1, or None for no
        top-k cut.  `trace` (list) receives the [1, V] logits of every step (tests).
        Sampling follows utils.py:102-157 in the reference's order.  The Exp(1) noise of its multinomial draw is the device stream
        of infer_panel_batch_infer (counter-based, seeded once per call from torch's CUDA generator), not torch.exponential_:
        torch.manual_seed still reproduces a run and greedy decoding does not depend on it, but sampled tokens differ from the
        reference's.
        Prompt-free decoding (prompts = None, TTS's ref_text_free mode; :796-803, :858-862): the prompt pass covers the text
        alone (full attention over it), the first logits come from the last text position, the token of step idx is embedded at
        pe[idx], and the result is (generated tokens without the last sample [1, n], 0); early_stop_num = 0 gives [1, 0].
        There is no CPU path: inputs that are not CUDA tensors raise NotImplementedError."""
        if not (x.is_cuda and bert_feature.is_cuda and (prompts is None or prompts.is_cuda)):
            raise NotImplementedError("infer_panel: decoding runs on CUDA tensors only (there is no CPU path)")
        assert x.shape[0] == 1 and (prompts is None or prompts.shape[0] == 1), "one utterance at a time, like infer_panel_naive"
        V = self.vocab_size
        if top_k is not None and (int(top_k) != top_k or top_k < 1):
            raise ValueError(f"infer_panel: top_k must be an integer >= 1 or None, got {top_k!r}")
        if int(max_steps) != max_steps or max_steps < 1:
            raise ValueError(f"infer_panel: max_steps must be an integer >= 1, got {max_steps!r}")
        ys, fin = self._decode_batch([x[0]], [x.shape[1]], [bert_feature[0]], prompts, x.shape[1], 11, int(max_steps),
                                     V if top_k is None else min(int(top_k), V), top_p, early_stop_num, temperature,
                                     repetition_penalty, trace)
        return ys[0][None], (0 if prompts is None else fin[0][0] - 1)

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
        inputs every row is decoded together (_decode_batch, text right-padded to max(kwargs["max_len"], longest row), which does
        not change the results); each row gives what infer_panel_naive(prompts=None) gives on it alone, up to the sampling noise:
        (y_list, [0] * B), y_list[b] the generated tokens without the last sample.  kwargs["trace"] (a list, tests) receives the
        raw [B, V] logits of every step.  Other inputs keep the per-row loop, which has no CPU path and raises
        NotImplementedError."""
        if prompts is None:
            self._check_ref_free(x, bert_feature, top_k)
            if all(t.is_cuda for t in list(x) + list(bert_feature)):
                lens = [int(x[b].shape[0]) for b in range(len(x))]
                max_len = max([int(kwargs.get("max_len", 0))] + lens)
                ys, _ = self._decode_batch(x, lens, bert_feature, None, max_len, 11, MAX_DECODE_STEPS, int(top_k), top_p,
                                           early_stop_num, temperature, repetition_penalty, kwargs.get("trace"))
                return ys, [0] * len(x)
        y_list, idx_list = [], []
        for i in range(len(x)):
            y, idx = self.infer_panel_naive(x[i].unsqueeze(0), x_lens[i], prompts[i].unsqueeze(0) if prompts is not None else None,
                                            bert_feature[i].unsqueeze(0), top_k, top_p, early_stop_num, temperature,
                                            repetition_penalty, **kwargs)
            y_list.append(y[0])
            idx_list.append(idx)
        return y_list, idx_list

    def _batch_state(self, dev, B, need_rows):
        """Per-layer caches [B, rows, 3 D] and the static buffers / graphs of the batched token step, kept across calls while the
        parameters, B and the capacity allow.  There are two: one for B = 1, its capacity rounded up to 512 rows so that single
        utterances of varying length rarely rebuild it, and one for B > 1, rounded up to 64 rows (a new B frees the previous one
        first).  Calls with one row and calls with several therefore do not rebuild each other's state."""
        ver = sum(int(p._version) for p in self.parameters())
        key, unit = ("_batch_st1", 512) if B == 1 else ("_batch_st", 64)
        st = self.__dict__.get(key)
        if st is not None and st["ver"] == ver and st["dev"] == dev and st["B"] == B and st["rows"] >= need_rows:
            return st
        self.__dict__.pop(key, None)
        rows = (need_rows + unit - 1) // unit * unit
        D, V, Vp = self.model_dim, self.vocab_size, (self.vocab_size + 3) // 4 * 4

        def z(*shape, dtype=torch.float32):
            return torch.zeros(shape, device=dev, dtype=dtype)
        st = dict(ver=ver, dev=dev, B=B, rows=rows, graphs={},
                  caches=[torch.empty((B, rows, 3 * D), device=dev, dtype=torch.float32) for _ in range(self.num_layers)],
                  n=z(1, dtype=torch.int32), x=z(B, 1, D), logits=z(B, Vp), skip=z(B, 2, dtype=torch.int32),
                  hist=z(B, rows, dtype=torch.int64), seen=z(B, (V + 31) // 32, dtype=torch.int32), fin=z(B, 2, dtype=torch.int32),
                  icfg=z(6, dtype=torch.int64), fcfg=z(3), pe=self.pe(rows, dev))
        self.__dict__[key] = st
        return st

    def _batch_step_graph(self, st, head, eos_steps):
        """The step graph of `st` whose sampler excludes EOS at the steps idx < eos_steps (a kernel argument, fixed at capture:
        1 for infer_panel_batch_infer, 11 for infer_panel_naive and prompt-free decoding), captured on first use."""
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

    def _run_batch(self, st, graph, prefix, n0, max_steps, top_k, early_stop_num, top_p, temperature, repetition_penalty, trace):
        """Decode every row of `st` (prompt pass done: caches, logits, n, skip, hist and seen set) until all have finished ->
        fin as a host list of [stop step, idx] per row.  The noise seed is drawn here, once per call, from torch's CUDA generator."""
        # one row reads the flags after every replay: a short utterance (~40 tokens) would otherwise run up to INFER_BATCH_K - 1
        # steps past its finish, which costs it more than the reads
        dev, K = st["dev"], (INFER_BATCH_K if st["B"] > 1 and trace is None else 1)
        st["fin"].fill_(-1)
        st["icfg"][0:1].copy_(torch.randint(0, 2 ** 62, (1,), device=dev, dtype=torch.int64))
        st["icfg"][1:].copy_(torch.tensor([prefix, n0, top_k, early_stop_num, max_steps], dtype=torch.int64))
        st["fcfg"].copy_(torch.tensor([float(top_p), float(temperature), float(repetition_penalty)], dtype=torch.float32))
        while True:
            for _ in range(K):
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
        Device path (_decode_batch): one prompt pass over [B, max_len + Yp] on the training kernels fills per-layer KV caches;
        then one CUDA graph per step (fused sampler + 24 layers of exact-fp32 row Linears and per-row-key decode attention +
        vocabulary projection) is replayed INFER_BATCH_K times between reads of the finished flags (once for a single row), so a
        batch has no per-token host sync.  Finished rows stay in the batch, frozen (the reference compacts them away; rows are independent, so the results
        are the same).  Batches of more than 64 rows run in chunks of 64.
        Random stream: the reference draws torch.exponential_ over a batch that shrinks as rows finish; here each Exp(1) draw is
        a counter-based function of (seed, row, step, token id) with the seed drawn once per call from torch's CUDA default
        generator, so torch.manual_seed still makes a run reproducible but sampled tokens differ from the reference's.
        Greedy decoding (top_k = 1) does not depend on the stream.  kwargs["trace"] (a list, tests) receives the raw [B, V]
        logits of every step and makes the host check the flags after every step."""
        if prompts is None:
            return self.infer_panel_naive_batched(x, x_lens, prompts, bert_feature, top_k=top_k, top_p=top_p,
                                                  early_stop_num=early_stop_num, temperature=temperature, **kwargs)
        B = len(x)
        V = self.vocab_size
        if int(top_k) != top_k or not 1 <= top_k <= V:
            raise ValueError(f"infer_panel_batch_infer: top_k must be an integer in [1, {V}], got {top_k!r}")
        top_k = int(top_k)
        if len(bert_feature) != B or prompts.dim() != 2 or prompts.shape[0] != B or len(x_lens) != B:
            raise ValueError("infer_panel_batch_infer: x, x_lens, prompts and bert_feature must have one entry per row")
        xl_host = [int(v) for v in x_lens]
        max_len = int(kwargs.get("max_len", max(xl_host)))
        for b in range(B):
            if x[b].dim() != 1 or bert_feature[b].shape != (1024, x[b].shape[0]) or not 1 <= xl_host[b] <= x[b].shape[0] <= max_len:
                raise ValueError(f"infer_panel_batch_infer: row {b}: x {tuple(x[b].shape)}, bert_feature {tuple(bert_feature[b].shape)}, "
                                 f"x_len {xl_host[b]}, max_len {max_len}")
        ys, fin = self._decode_batch(x, xl_host, bert_feature, prompts, max_len, 1, MAX_DECODE_STEPS, top_k, top_p, early_stop_num,
                                     temperature, repetition_penalty, kwargs.get("trace"))
        return ys, [f[1] for f in fin]

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
    def _decode_batch(self, rows, lens, bert, prompts, max_len, eos_steps, max_steps, top_k, top_p, early_stop_num, temperature,
                      repetition_penalty, trace):
        """The KV-cache decoder behind every public decoding method: all rows decoded together -> (hist slices, fin), slice b the
        1-D int64 prompt + generated tokens of row b (hist[b, :Yp + fin[b][0]]), fin[b] its [stop step, idx] (evk_sample_tokens).
        The callers check the arguments: rows[b] is 1-D, at most max_len wide, and its first lens[b] positions are text; bert[b]
        is [1024, rows[b] width]; prompts is [B, Yp] or None (Yp = 0); top_k lies in [1, V]; max_steps >= 1.
          - Prompt pass: one pass over [B, max_len + Yp] on the training kernels (text right-padded to max_len; ragged prefix-LM
            flash attention with xlen = lens, ylen = Yp) fills per-layer caches of in_proj rows.  Row b's first logits come from
            position max_len + Yp - 1 (its last prompt token) with a prompt, from its last text position lens[b] - 1 without.
          - Step idx (_run_batch, one replay of the step graph): the token goes to cache row max_len + Yp + idx and is embedded
            at pe[Yp + idx] (:705, :858-859); each row leaves out its text padding lens[b] .. max_len - 1; EOS is excluded at the
            steps idx < eos_steps; a row stops when its sample or the argmax of its penalised logits is EOS (fin (idx, idx - 1)),
            or at idx + 1 > early_stop_num (!= -1) or idx == max_steps - 1 (fin (idx, idx)).
        The caches hold max_len + Yp + min(max_steps, early_stop_num + 1) + INFER_BATCH_K rows of 3 * 512 floats per layer and
        row (_batch_state rounds this up): 24 layers x B x rows x 6 KiB, e.g. 1.4 GiB for B = 16, max_len 120, Yp 150,
        early_stop_num 300 (640 rows).  Batches of more than 64 rows run in chunks of 64 (the row Linears take 64 rows per
        launch).  `trace` (a list, tests) receives the raw [B, V] logits of every step."""
        B = len(rows)
        if B > 64:
            out = [self._decode_batch(rows[i:i + 64], lens[i:i + 64], bert[i:i + 64], None if prompts is None else prompts[i:i + 64],
                                      max_len, eos_steps, max_steps, top_k, top_p, early_stop_num, temperature, repetition_penalty,
                                      trace)
                   for i in range(0, B, 64)]
            return [y for o in out for y in o[0]], [f for o in out for f in o[1]]
        dev = (rows[0] if prompts is None else prompts).device
        Yp = 0 if prompts is None else prompts.shape[1]
        L0 = max_len + Yp
        cap = max_steps if early_stop_num == -1 else min(max_steps, early_stop_num + 1)
        was_training = self.training
        self.eval()
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            xp = torch.zeros((B, max_len), device=dev, dtype=torch.int64)
            bp = torch.zeros((B, 1024, max_len), device=dev, dtype=torch.float32)
            for b in range(B):
                xp[b, :rows[b].shape[0]] = rows[b]
                bp[b, :, :rows[b].shape[0]] = bert[b]
            st = self._batch_state(dev, B, L0 + cap + INFER_BATCH_K)
            Vp = st["logits"].shape[1]
            head = self.w("ar_predict_layer", pad0=Vp)
            graph = self._batch_step_graph(st, head, eos_steps)
            # prompt pass (process_prompt with the padded mask, :596-646; prompt-free: the text alone, :796-803)
            y = torch.zeros((B, 0), device=dev, dtype=torch.int64) if prompts is None else prompts.to(torch.int64)
            xe = self._embed_text(xp, bp, False)
            ye = ops.embedding(self.P("ar_audio_embedding.word_embeddings.weight"), y)
            h = ops.gpt_embed(xe, ye, self.P("ar_text_position.alpha"), self.P("ar_audio_position.alpha"), st["pe"])
            xl = torch.tensor(lens, device=dev, dtype=torch.int64)
            yl = torch.full((B,), Yp, device=dev, dtype=torch.int64)
            for i in range(self.num_layers):
                h = self._infer_layer(i, h, st["caches"][i], None, X=max_len, xl=xl, yl=yl)
            first = xl - 1 if prompts is None else torch.full((B,), L0 - 1, device=dev, dtype=torch.int64)
            st["logits"].copy_(ops.linear_rows(ops.slice_rows(h, first, 1), head).view(B, Vp))
            # per-call state of the step graph
            st["n"].fill_(L0)
            st["skip"].copy_(torch.tensor([[v, max_len] for v in lens], dtype=torch.int32))
            st["hist"][:, :Yp].copy_(y)
            bits = torch.zeros((B, st["seen"].shape[1] * 32), device=dev, dtype=torch.int64).scatter_(1, y, 1)
            words = (bits.view(B, -1, 32) << torch.arange(32, device=dev, dtype=torch.int64)).sum(-1)
            st["seen"].copy_(torch.where(words >= 2 ** 31, words - 2 ** 32, words))      # uint32 bit patterns as int32
            fin = self._run_batch(st, graph, Yp, L0, max_steps, top_k, early_stop_num, top_p, temperature, repetition_penalty, trace)
            return [st["hist"][b, :Yp + fin[b][0]].clone() for b in range(B)], fin
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
