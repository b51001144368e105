"""Stage-2 networks: SynthesizerTrn (SoVITS acoustic model + HiFi-GAN generator) and MultiPeriodDiscriminator.

Same constructor arguments, forward signatures and ``state_dict()`` keys/shapes as the reference
(the reference's src/easevoice/module/models.py:803-946, 590-614), but every tensor operation is a libevk_sm90
kernel on channels-last activations.  ``forward`` keeps the reference's [B, C, T] contract at the API boundary;
``forward_cl`` is the channels-last fast path the trainer uses.

Randomness is injectable (``noise``, ``ids_slice``) for parity tests; when omitted it is drawn on the device
from the library's Philox streams (no host sync, CUDA-graph safe).  Dropout follows ``self.training`` like the
reference (p_dropout for enc_p, 0.1 inside MelStyleEncoder).
"""
import math
import contextlib
import os

import torch
from torch import nn

from . import lib, ops

D_LANES = max(1, min(6, int(os.environ.get("EVK_D_LANES", "6"))))   # streams the six discriminators are spread over
D_PRIO = os.environ.get("EVK_D_PRIO", "0") == "1"                    # DiscriminatorS on a high-priority stream (experiment)
SIDE_STREAMS = os.environ.get("EVK_SIDE_STREAMS", "1") != "0"     # prior encoder on a side stream (measured 66.5 -> 63.0 ms / step)
LRELU_SLOPE = 0.1
N_SYMBOLS = 732            # len(SYMBOLS): src/easevoice/text/symbols.py:410-412
PERIODS = (2, 3, 5, 7, 11)


class _Node(nn.Module):
    pass


class ParamTree(nn.Module):
    """nn.Module whose parameters/buffers are registered under dotted reference names."""

    def _register(self, name, tensor, buffer=False):
        node = self
        parts = name.split(".")
        for p in parts[:-1]:
            if not hasattr(node, p):
                node.add_module(p, _Node())
            node = getattr(node, p)
        if buffer:
            node.register_buffer(parts[-1], tensor)
        else:
            node.register_parameter(parts[-1], nn.Parameter(tensor))

    def P(self, name):
        node = self
        for p in name.split("."):
            node = getattr(node, p)
        return node

    def has(self, name):
        node = self
        for p in name.split("."):
            if not hasattr(node, p):
                return False
            node = getattr(node, p)
        return True

    def _side_stream(self, device, idx=0, priority=0):
        key = f"_side{idx}"
        st = self.__dict__.get(key)
        if st is None or st.device != device:
            st = torch.cuda.Stream(device=device, priority=priority)
            self.__dict__[key] = st
        return st

    # ---- packed-weight helpers (weight-norm folded into the packing pass) --------------------
    _frozen = False            # True: weights enter the graph as constants (no weight gradients are computed)

    def begin_pack(self):
        """Call at the start of a forward pass.  The first pass of each kind (frozen or not) packs layer by layer and records
        what it packs; later passes run the recorded plan in one launch and hand out views of its arenas.  Inference
        without gradients on a network that is not frozen packs layer by layer on use."""
        self._active, self._recording = None, None
        if not torch.is_grad_enabled() and not self._frozen:
            return
        plans = self.__dict__.setdefault("_plans", {})
        plan = plans.get(self._frozen)
        if plan is not None and not plan.valid():
            plan = plans.pop(self._frozen, None) and None
        if plan is None:
            self._recording = []
            return
        packed = ops.pack_all(plan)
        self._active = {req[0]: pw for req, pw in zip(plan.reqs, packed)}

    def end_pack(self):
        rec, self._recording, self._active = getattr(self, "_recording", None), None, None
        if rec:
            self.__dict__.setdefault("_plans", {})[self._frozen] = ops.PackPlan(rec, with_grad=not self._frozen)

    def w(self, pfx, need_pb=True, pad0=0, pad1=0, suffix=".weight"):
        """packed (and weight-normed when pfx has weight_g / weight_v) operand of the parameter `pfx + suffix`"""
        key = (pfx, need_pb, pad0, pad1)
        act = getattr(self, "_active", None)
        if act is not None and key in act:
            return act[key]
        fz = (lambda t: t.detach()) if self._frozen else (lambda t: t)
        has_g = self.has(pfx + ".weight_v")
        v = self.P(pfx + (".weight_v" if has_g else suffix))
        g = self.P(pfx + ".weight_g") if has_g else None
        rec = getattr(self, "_recording", None)
        if rec is not None and all(r[0] != key for r in rec):
            rec.append((key, v, g, need_pb, pad0, pad1, torch.is_grad_enabled() and not self._frozen))
        pw = ops.pack_weight(fz(v), fz(g) if g is not None else None, need_pb, pad0, pad1)
        if act is not None and getattr(self, "_memo_pack", False):
            act[key] = pw                      # inference: static weights are packed once and kept (see inference_weights)
        return pw

    def weights_key(self):
        """What packed operands, and CUDA graphs captured with them, depend on: the parameters' and buffers' version counters,
        the device, and the precise mode (pack_weight rounds to TF32 unless evk_set_precise(1) is on, and a graph replays the
        kernels of the mode it was captured in)."""
        # one walk over the modules: parameters() and buffers() together take two to three times as long
        ver = sum(t._version for m in self.modules() for t in (*m._parameters.values(), *m._buffers.values()) if t is not None)
        return ver, str(next(self.parameters()).device), lib.load().evk_get_precise()

    def cached(self, name, build):
        """build()'s result, kept under `name` until weights_key() changes."""
        key = self.weights_key()
        cache = self.__dict__.setdefault("_cached", {})
        if name not in cache or cache[name][0] != key:
            cache.pop(name, None)              # free the stale value before its replacement is built
            cache[name] = (key, build())
        return cache[name][1]

    def packed_for_inference(self):
        """-> the dict inference_weights() hands to w() as `self._active`: the packed weights made during inference, kept until
        weights_key() changes."""
        return self.cached("inference", dict)

    @contextlib.contextmanager
    def inference_weights(self):
        """Scope of an inference pass: every packed weight w() makes is kept (packed_for_inference) and handed out again by later
        passes."""
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            yield
        finally:
            self._active, self._memo_pack = None, False

    def b(self, pfx, pad=0):
        if not self.has(pfx + ".bias"):
            return None
        b = self.P(pfx + ".bias")
        if self._frozen:
            b = b.detach()
        if pad > b.shape[0]:
            b = torch.nn.functional.pad(b, (0, pad - b.shape[0]))
        return b


def _kaiming_uniform_(t, fan_in, gen):
    bound = 1.0 / math.sqrt(fan_in) if fan_in > 0 else 0.0
    with torch.no_grad():
        t.copy_((torch.rand(t.shape, generator=gen) * 2 - 1) * bound)


# ====================================================================================================
# SynthesizerTrn
# ====================================================================================================
class SynthesizerTrn(ParamTree):
    """models.py:803-946."""

    def __init__(self, spec_channels, segment_size, inter_channels, hidden_channels, filter_channels, n_heads, n_layers,
                 kernel_size, p_dropout, resblock, resblock_kernel_sizes, resblock_dilation_sizes, upsample_rates,
                 upsample_initial_channel, upsample_kernel_sizes, n_speakers=0, gin_channels=0, use_sdp=True,
                 semantic_frame_rate=None, freeze_quantizer=None, version="v2", **kwargs):
        super().__init__()
        assert resblock == "1" and semantic_frame_rate == "25hz" and version == "v2" and gin_channels > 0
        self.spec_channels, self.segment_size = spec_channels, segment_size
        self.inter_channels, self.hidden_channels, self.filter_channels = inter_channels, hidden_channels, filter_channels
        self.n_heads, self.n_layers, self.kernel_size, self.p_dropout = n_heads, n_layers, kernel_size, p_dropout
        self.resblock_kernel_sizes, self.resblock_dilation_sizes = resblock_kernel_sizes, resblock_dilation_sizes
        self.upsample_rates, self.upsample_kernel_sizes = upsample_rates, upsample_kernel_sizes
        self.upsample_initial_channel, self.gin_channels = upsample_initial_channel, gin_channels
        self.freeze_quantizer = freeze_quantizer
        self._cb_inited = None         # (version counter, value) of the codebook's `inited` flag (codebook_needs_init)
        self.window = 4
        self.style_dropout = 0.1
        self._build()
        self.reset_parameters()

    # ------------------------------------------------------------------------------------------
    def _conv(self, name, cout, cin, k, bias=True, wn=False):
        if wn:
            self._register(name + ".bias", torch.zeros(cout)) if bias else None
            self._register(name + ".weight_g", torch.ones(cout, 1, 1))
            self._register(name + ".weight_v", torch.zeros(cout, cin, k))
        else:
            self._register(name + ".weight", torch.zeros(cout, cin, k))
            if bias:
                self._register(name + ".bias", torch.zeros(cout))

    def _encoder(self, pfx, n_layers):
        H, F, k, dk = self.hidden_channels, self.filter_channels, self.kernel_size, self.hidden_channels // self.n_heads
        for i in range(n_layers):
            a = f"{pfx}.attn_layers.{i}"
            self._register(a + ".emb_rel_k", torch.zeros(1, 2 * self.window + 1, dk))
            self._register(a + ".emb_rel_v", torch.zeros(1, 2 * self.window + 1, dk))
            for c in "qkvo":
                self._conv(f"{a}.conv_{c}", H, H, 1)
            self._register(f"{pfx}.norm_layers_1.{i}.gamma", torch.ones(H))
            self._register(f"{pfx}.norm_layers_1.{i}.beta", torch.zeros(H))
            self._conv(f"{pfx}.ffn_layers.{i}.conv_1", F, H, k)
            self._conv(f"{pfx}.ffn_layers.{i}.conv_2", H, F, k)
            self._register(f"{pfx}.norm_layers_2.{i}.gamma", torch.ones(H))
            self._register(f"{pfx}.norm_layers_2.{i}.beta", torch.zeros(H))

    def _wn(self, pfx, k, n_layers):
        H, gin = self.hidden_channels, self.gin_channels
        # registration order = the reference's named_parameters() order (modules.py:153-185: in/res_skip ModuleLists are
        # assigned before cond_layer), so optimizer state indices line up with torch.optim.AdamW checkpoints
        for i in range(n_layers):
            self._conv(f"{pfx}.in_layers.{i}", 2 * H, H, k, wn=True)
        for i in range(n_layers):
            self._conv(f"{pfx}.res_skip_layers.{i}", 2 * H if i < n_layers - 1 else H, H, 1, wn=True)
        self._conv(pfx + ".cond_layer", 2 * H * n_layers, gin, 1, wn=True)

    def _build(self):
        H, I, gin = self.hidden_channels, self.inter_channels, self.gin_channels
        # enc_p
        self._conv("enc_p.ssl_proj", H, 768, 1)
        self._encoder("enc_p.encoder_ssl", self.n_layers // 2)
        self._encoder("enc_p.encoder_text", self.n_layers)
        self._register("enc_p.text_embedding.weight", torch.zeros(N_SYMBOLS, H))
        for c in "qkvo":
            self._conv(f"enc_p.mrte.cross_attention.conv_{c}", 512, 512, 1)
        self._conv("enc_p.mrte.c_pre", 512, H, 1)
        self._conv("enc_p.mrte.text_pre", 512, H, 1)
        self._conv("enc_p.mrte.c_post", H, 512, 1)
        self._encoder("enc_p.encoder2", self.n_layers // 2)
        self._conv("enc_p.proj", 2 * I, H, 1)
        # dec
        C0 = self.upsample_initial_channel
        self._conv("dec.conv_pre", C0, I, 7)
        for i, (u, k) in enumerate(zip(self.upsample_rates, self.upsample_kernel_sizes)):
            cin, cout = C0 // 2 ** i, C0 // 2 ** (i + 1)
            self._register(f"dec.ups.{i}.bias", torch.zeros(cout))
            self._register(f"dec.ups.{i}.weight_g", torch.ones(cin, 1, 1))
            self._register(f"dec.ups.{i}.weight_v", torch.zeros(cin, cout, k))
        nk = len(self.resblock_kernel_sizes)
        for i in range(len(self.upsample_rates)):
            ch = C0 // 2 ** (i + 1)
            for j, k in enumerate(self.resblock_kernel_sizes):
                for grp in ("convs1", "convs2"):
                    for l in range(3):
                        self._conv(f"dec.resblocks.{i * nk + j}.{grp}.{l}", ch, ch, k, wn=True)
        self._conv("dec.conv_post", 1, C0 // 2 ** len(self.upsample_rates), 7, bias=False)
        self._conv("dec.cond", C0, gin, 1)
        # enc_q / flow
        self._conv("enc_q.pre", H, self.spec_channels, 1)
        self._wn("enc_q.enc", 5, 16)
        self._conv("enc_q.proj", 2 * I, H, 1)
        for f in range(4):
            p = f"flow.flows.{2 * f}"
            self._conv(p + ".pre", H, I // 2, 1)
            self._wn(p + ".enc", 5, 4)
            self._conv(p + ".post", I // 2, H, 1)
        # ref_enc
        self._register("ref_enc.spectral.0.fc.weight", torch.zeros(128, 704))
        self._register("ref_enc.spectral.0.fc.bias", torch.zeros(128))
        self._register("ref_enc.spectral.3.fc.weight", torch.zeros(128, 128))
        self._register("ref_enc.spectral.3.fc.bias", torch.zeros(128))
        for i in range(2):
            self._register(f"ref_enc.temporal.{i}.conv1.conv.weight", torch.zeros(256, 128, 5))
            self._register(f"ref_enc.temporal.{i}.conv1.conv.bias", torch.zeros(256))
        for n in ("w_qs", "w_ks", "w_vs", "fc"):
            self._register(f"ref_enc.slf_attn.{n}.weight", torch.zeros(128, 128))
            self._register(f"ref_enc.slf_attn.{n}.bias", torch.zeros(128))
        self._register("ref_enc.fc.fc.weight", torch.zeros(gin, 128))
        self._register("ref_enc.fc.fc.bias", torch.zeros(gin))
        # top level
        self._conv("ssl_proj", 768, 768, 2)
        cb = "quantizer.vq.layers.0._codebook."
        self._register(cb + "inited", torch.ones(1), buffer=True)
        self._register(cb + "cluster_size", torch.zeros(1024), buffer=True)
        self._register(cb + "embed", torch.zeros(1024, 768), buffer=True)
        self._register(cb + "embed_avg", torch.zeros(1024, 768), buffer=True)

    def reset_parameters(self, seed=1234):
        """Random init with the reference's distributions (used when no pretrained checkpoint is given)."""
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.endswith("weight_v"):
                    if name.startswith("dec."):
                        p.copy_(torch.randn(p.shape, generator=g) * 0.01)     # commons.init_weights
                    else:
                        _kaiming_uniform_(p, p[0].numel(), g)
                elif name.endswith((".gamma",)):
                    p.fill_(1.0)
                elif name.endswith((".beta",)):
                    p.zero_()
                elif "emb_rel" in name:
                    p.copy_(torch.randn(p.shape, generator=g) * p.shape[-1] ** -0.5)
                elif name.endswith("text_embedding.weight"):
                    p.copy_(torch.randn(p.shape, generator=g))
                elif name.endswith(".weight"):
                    _kaiming_uniform_(p, p[0].numel(), g)
                elif name.endswith(".bias"):
                    base = name[:-4]
                    wname = base + ("weight_v" if self.has(base + "weight_v") else "weight")
                    _kaiming_uniform_(p, self.P(wname)[0].numel(), g)
            for name, p in self.named_parameters():
                if name.endswith("weight_g"):                                  # weight_norm: g = ||v||
                    v = self.P(name[:-1] + "v")
                    p.copy_(v.flatten(1).norm(dim=1).view(p.shape))
            for f in range(4):                                                  # modules.py:436-437
                self.P(f"flow.flows.{2 * f}.post.weight").zero_()
                self.P(f"flow.flows.{2 * f}.post.bias").zero_()
            cb = "quantizer.vq.layers.0._codebook."
            emb = self.P(cb + "embed")
            emb.copy_(torch.randn(emb.shape, generator=g))
            self.P(cb + "embed_avg").copy_(emb)
            if self.freeze_quantizer is False:
                # a fresh reference quantizer (kmeans_init=True, core_vq.py:124-138): zero codebook, k-means on the first batch
                for n in ("embed", "embed_avg", "cluster_size", "inited"):
                    self.P(cb + n).zero_()

    # ---------------------------------------------------------------------------------------------
    # blocks (channels-last)
    # ---------------------------------------------------------------------------------------------
    def _attn_encoder(self, pfx, x, length, n_layers):
        """attentions.py:67-90."""
        H = self.n_heads
        dk = self.hidden_channels // H
        p = self.p_dropout if self.training else 0.0
        pad = self.kernel_size // 2
        x = ops.rowmask(x, length)
        for i in range(n_layers):
            a = f"{pfx}.attn_layers.{i}"
            q = ops.linear(x, self.w(a + ".conv_q"), self.b(a + ".conv_q"))
            k = ops.linear(x, self.w(a + ".conv_k"), self.b(a + ".conv_k"))
            v = ops.linear(x, self.w(a + ".conv_v"), self.b(a + ".conv_v"))
            o = ops.attention(q, k, v, heads=H, scale=1.0 / math.sqrt(dk), Ek=self.P(a + ".emb_rel_k"),
                              Ev=self.P(a + ".emb_rel_v"), window=self.window, fill=-1e4, qlen=length, klen=length,
                              p_drop=p, tag=a + ".drop")
            y = ops.linear(o, self.w(a + ".conv_o"), self.b(a + ".conv_o"))
            y = ops.dropout(y, p, a + ".odrop")
            x = ops.layernorm(x, self.P(f"{pfx}.norm_layers_1.{i}.gamma"), self.P(f"{pfx}.norm_layers_1.{i}.beta"), res=y)
            # FFN(x * mask) (attentions.py:408-416): rows past `length` never influence valid rows (keys are masked, every
            # conv input is masked), so the stream itself is masked here once and both convs run without an input mask
            # (unmasked launches are the ones the TMA/wgmma kernel takes); conv_1's epilogue mask == masking conv_2's input
            x = ops.rowmask(x, length)
            f = f"{pfx}.ffn_layers.{i}"
            h = ops.conv(x, self.w(f + ".conv_1"), self.b(f + ".conv_1"), pad=pad, act=ops.ACT_RELU, out_len=length)
            h = ops.dropout(h, p, f + ".drop1")
            h = ops.conv(h, self.w(f + ".conv_2"), self.b(f + ".conv_2"), pad=pad, out_len=length)
            h = ops.dropout(h, p, f + ".drop2")
            x = ops.layernorm(x, self.P(f"{pfx}.norm_layers_2.{i}.gamma"), self.P(f"{pfx}.norm_layers_2.{i}.beta"), res=h)
        return ops.rowmask(x, length)

    def _wn_stack(self, pfx, x, length, g, n_layers, k=5):
        """modules.py:187-212 (dilation_rate 1, p_dropout 0)."""
        H = self.hidden_channels
        cond = ops.linear(g, self.w(pfx + ".cond_layer"), self.b(pfx + ".cond_layer"))        # [B, 1, 2H*n]
        out = None
        for i in range(n_layers):
            a = ops.conv(x, self.w(f"{pfx}.in_layers.{i}"), self.b(f"{pfx}.in_layers.{i}"), pad=(k - 1) // 2)
            acts = ops.wn_gate(a, cond[:, :, i * 2 * H:(i + 1) * 2 * H])
            rs = ops.linear(acts, self.w(f"{pfx}.res_skip_layers.{i}"), self.b(f"{pfx}.res_skip_layers.{i}"))
            if i < n_layers - 1:
                x = ops.add(x, rs[:, :, :H], length=length)
                skip = rs[:, :, H:]
            else:
                skip = rs
            out = skip if out is None else ops.add(out, skip)
        return ops.rowmask(out, length)

    def _ref_enc(self, spec, length):
        """MelStyleEncoder, modules.py:739-763.  spec [B, T, 1025] -> ge [B, 1, 512]."""
        pfx = "ref_enc"
        p = self.style_dropout if self.training else 0.0
        x = ops.rowmask(spec[:, :, :704], length)                                # y * y_mask (models.py:906-909)
        x = ops.linear(x, self.w(pfx + ".spectral.0.fc"), self.b(pfx + ".spectral.0.fc"))
        x = ops.dropout(ops.mish(x), p, pfx + ".d0")
        x = ops.linear(x, self.w(pfx + ".spectral.3.fc"), self.b(pfx + ".spectral.3.fc"))
        x = ops.dropout(ops.mish(x), p, pfx + ".d1")
        for i in range(2):
            c = f"{pfx}.temporal.{i}.conv1.conv"
            h = ops.conv(x, self.w(c), self.b(c), pad=2)
            if p > 0.0:
                x = ops.add(x, ops.dropout(ops.glu_res(None, h), p, f"{pfx}.g{i}"))
            else:
                x = ops.glu_res(x, h)
        x = ops.rowmask(x, length)
        a = pfx + ".slf_attn"
        q = ops.linear(x, self.w(a + ".w_qs"), self.b(a + ".w_qs"))
        k = ops.linear(x, self.w(a + ".w_ks"), self.b(a + ".w_ks"))
        v = ops.linear(x, self.w(a + ".w_vs"), self.b(a + ".w_vs"))
        o = ops.attention(q, k, v, heads=2, scale=1.0 / math.sqrt(128.0), fill=float("-inf"), klen=length, p_drop=p,
                          tag=a + ".drop")
        o = ops.linear(o, self.w(a + ".fc"), self.b(a + ".fc"))
        x = ops.add(ops.dropout(o, p, a + ".odrop"), x)
        x = ops.linear(x, self.w(pfx + ".fc.fc"), self.b(pfx + ".fc.fc"))
        return ops.masked_mean(x, length).unsqueeze(1)

    def _enc_p(self, quantized, length, text, text_len, ge, speed=1):
        """TextEncoder.forward, models.py:228-251.  speed != 1 (inference only, models.py:246-248): the encoder output is
        resampled linearly to int(T / speed) + 1 frames before the projection; returns (stats, new_length) in that case."""
        y = ops.linear(ops.rowmask(quantized, length), self.w("enc_p.ssl_proj"), self.b("enc_p.ssl_proj"), out_len=length)
        y = self._attn_encoder("enc_p.encoder_ssl", y, length, self.n_layers // 2)
        t = ops.embedding(self.P("enc_p.text_embedding.weight"), text)
        t = self._attn_encoder("enc_p.encoder_text", t, text_len, self.n_layers)
        # MRTE, mrte_model.py:25-61
        m = "enc_p.mrte"
        # y and t leave _attn_encoder masked; c_pre / text_pre mask their OUTPUT in the epilogue, which is the masked input
        # the cross attention reads (mrte_model.py:52-58); only rows past `length` differ from the reference (they are
        # masked again before c_post), so every Linear here is an unmasked TMA launch
        ssl_enc = ops.linear(y, self.w(m + ".c_pre"), self.b(m + ".c_pre"), out_len=length)
        text_enc = ops.linear(t, self.w(m + ".text_pre"), self.b(m + ".text_pre"), out_len=text_len)
        ca = m + ".cross_attention"
        q = ops.linear(ssl_enc, self.w(ca + ".conv_q"), self.b(ca + ".conv_q"))
        k = ops.linear(text_enc, self.w(ca + ".conv_k"), self.b(ca + ".conv_k"))
        v = ops.linear(text_enc, self.w(ca + ".conv_v"), self.b(ca + ".conv_v"))
        a = ops.attention(q, k, v, heads=4, scale=1.0 / math.sqrt(128.0), fill=-1e4, qlen=length, klen=text_len)
        a = ops.linear(a, self.w(ca + ".conv_o"), self.b(ca + ".conv_o"))
        x = ops.rowmask(ops.add_bvec(ops.add(a, ssl_enc), ge), length)
        y = ops.linear(x, self.w(m + ".c_post"), self.b(m + ".c_post"))
        y = self._attn_encoder("enc_p.encoder2", y, length, self.n_layers // 2)
        if speed != 1:
            # F.interpolate(y, size, mode="linear") along time, and the (all-ones) mask by nearest: rows are full length here
            # because decode() runs one utterance at a time (y_lengths = [2T], models.py:995)
            assert bool((length == y.shape[1]).all()), "speed != 1 needs unpadded rows"
            Tn = int(y.shape[1] / speed) + 1
            y = torch.nn.functional.interpolate(y.transpose(1, 2), size=Tn, mode="linear").transpose(1, 2).contiguous()
            length = torch.full_like(length, Tn)
            return ops.linear(y, self.w("enc_p.proj"), self.b("enc_p.proj"), out_len=length), length
        stats = ops.linear(y, self.w("enc_p.proj"), self.b("enc_p.proj"), out_len=length)
        return stats

    def _generator(self, z, ge, lengths=None):
        """Generator.forward, models.py:452-471 + ResBlock1 modules.py:298-311.  lengths (inference, int32 device [B], frames
        of z; z zero past them): rows of different lengths.  Every conv then writes zeros past the row's length at its rate, so
        every conv reads zeros there, as it reads the zero padding past the end of a row vocoded alone."""
        lens = lengths
        x = ops.conv(z, self.w("dec.conv_pre"), self.b("dec.conv_pre"), pad=3, out_len=lens)
        x = ops.add_bvec(x, ops.linear(ge, self.w("dec.cond"), self.b("dec.cond")))
        if lens is not None:
            x = ops.rowmask(x, lens)                       # the conditioning vector is added to every row
        nk = len(self.resblock_kernel_sizes)
        for i, (u, k) in enumerate(zip(self.upsample_rates, self.upsample_kernel_sizes)):
            x = ops.lrelu(x, LRELU_SLOPE)
            lens = None if lens is None else lens * u
            x = ops.conv_transpose(x, self.w(f"dec.ups.{i}"), self.b(f"dec.ups.{i}"), stride=u, pad=(k - u) // 2, out_len=lens)
            xa = ops.lrelu(x, LRELU_SLOPE)                 # shared first activation of the three resblocks
            outs = []
            # the three resblocks of a stage are independent chains of six convolutions; stage 0 is 40 tiles on 132 SMs and
            # stage 1 is 2.16 waves of the persistent grid, so they run as three parallel branches (streams 2, 3 + current;
            # 0 and 1 may still be busy with the prior encoder and the flow)
            cur = torch.cuda.current_stream() if (SIDE_STREAMS and x.is_cuda) else None
            lanes = [None, self._side_stream(x.device, 2), self._side_stream(x.device, 3)] if cur is not None and nk == 3 else [None] * nk
            for j, (rk, rd) in enumerate(zip(self.resblock_kernel_sizes, self.resblock_dilation_sizes)):
                r = f"dec.resblocks.{i * nk + j}"
                st = lanes[j]
                if st is not None:
                    st.wait_stream(cur)
                    x.record_stream(st); xa.record_stream(st)
                with (torch.cuda.stream(st) if st is not None else contextlib.nullcontext()):
                    h, ha = x, xa
                    for l, d in enumerate(rd):
                        t = ops.conv(ha, self.w(f"{r}.convs1.{l}"), self.b(f"{r}.convs1.{l}"), pad=(rk * d - d) // 2, dil=d,
                                     act=ops.ACT_LRELU, slope=LRELU_SLOPE, out_len=lens)
                        h = ops.conv(t, self.w(f"{r}.convs2.{l}"), self.b(f"{r}.convs2.{l}"), pad=(rk - 1) // 2, res=h,
                                     out_len=lens)
                        if l < len(rd) - 1:
                            ha = ops.lrelu(h, LRELU_SLOPE)
                if st is not None:
                    h.record_stream(cur)
                outs.append(h)
            for st in lanes:
                if st is not None:
                    cur.wait_stream(st)
            x = ops.add3(outs[0], outs[1], outs[2], 1.0 / nk, 1.0 / nk, 1.0 / nk)
        x = ops.lrelu(x, 0.01)                             # F.leaky_relu default slope (models.py:467)
        # the single output channel is padded to 4 (zero weights) so that its gradients stay on the tensor-core kernels
        y4 = ops.conv(x, self.w("dec.conv_post", pad0=4), None, pad=3, act=ops.ACT_TANH, out_len=lens)
        return ops.take_channels(y4, 1)

    # ---------------------------------------------------------------------------------------------
    def _flow(self, z, lengths, ge):
        I = self.inter_channels
        zf, half = z, I // 2
        for f in range(4):
            p = f"flow.flows.{2 * f}"
            x0, x1 = zf[:, :, :half], zf[:, :, half:]
            h = ops.linear(x0, self.w(p + ".pre"), self.b(p + ".pre"), out_len=lengths)
            h = self._wn_stack(p + ".enc", h, lengths, ge, 4)
            m = ops.linear(h, self.w(p + ".post"), self.b(p + ".post"), out_len=lengths)
            x1 = ops.add(m, x1, length=lengths)
            zf = ops.cat_flip(x0, x1)
        return zf

    def forward_cl(self, ssl, spec, lengths, text, text_lengths, noise=None, ids_slice=None, vq_rows=None, kmeans_idx=None):
        """Channels-last forward.  ssl [B,T,768], spec [B,T,1025] (pitch may be padded), lengths/text_lengths int32 [B],
        text int64 [B,X].  Returns a dict of channels-last tensors (same quantities as SynthesizerTrn.forward).
        Trainable quantizer only: vq_rows (device int32 [1]) is the reference collate's frame count / 2, so that rows
        past it (padding to a coarser grid) take no part in the codebook statistics or the commitment loss (default:
        all T / 2 rows); kmeans_idx (int64 [1024]) replaces the random draw of the k-means initial means."""
        self.begin_pack()
        try:
            return self._forward_cl(ssl, spec, lengths, text, text_lengths, noise, ids_slice, vq_rows, kmeans_idx)
        finally:
            self.end_pack()

    @property
    def quantizer_trainable(self):
        """freeze_quantizer: false (only an explicit False; None keeps the frozen path) and training mode."""
        return self.freeze_quantizer is False and self.training

    def codebook_needs_init(self):
        """Host-side: does the next trainable-quantizer forward k-means-initialise the codebook (inited == 0)?  Reads the
        device buffer (a synchronisation) only when it was written from PyTorch since the last read (checkpoint loads)."""
        inited = self.P("quantizer.vq.layers.0._codebook.inited")
        if self._cb_inited is None or self._cb_inited[0] != inited._version:
            assert not (inited.is_cuda and torch.cuda.is_current_stream_capturing()), "codebook state must be known before capture"
            self._cb_inited = (inited._version, bool(inited.item() != 0))
        return not self._cb_inited[1]

    def _quantize_train(self, ssl, vq_rows, kmeans_idx):
        """VectorQuantization.forward in training mode (core_vq.py:203-228, 301-318): k-means init when inited == 0,
        codes from the (new) codebook, EMA update of the buffers, straight-through value and commitment loss.
        -> (quantized [B, T, 768], codes [B, T/2], commit loss)."""
        cb = "quantizer.vq.layers.0._codebook."
        embed, embed_avg = self.P(cb + "embed"), self.P(cb + "embed_avg")
        cluster_size, inited = self.P(cb + "cluster_size"), self.P(cb + "inited")
        x = ops.ssl_proj_fp32(ssl, self.P("ssl_proj.weight"), self.P("ssl_proj.bias"))      # [B, T/2, 768], exact fp32
        if vq_rows is None:
            vq_rows = torch.full((1,), x.shape[1], device=x.device, dtype=torch.int32)
        with torch.no_grad():
            if self.codebook_needs_init():
                ops.vq_kmeans_init_(x, vq_rows, embed, embed_avg, cluster_size, inited, idx=kmeans_idx)
                self._cb_inited = (inited._version, True)
            codes = ops.vq_nearest(x, embed)
            q = ops.embedding(embed, codes)                  # looked up before the EMA overwrites embed (core_vq.py:209-226)
            ops.vq_ema_(x, codes, vq_rows, cluster_size, embed_avg, embed)
        quantized, commit = ops.vq_straight_through(x, q, vq_rows)
        return quantized, codes, commit

    def _forward_cl(self, ssl, spec, lengths, text, text_lengths, noise, ids_slice, vq_rows=None, kmeans_idx=None):
        B, T, _ = spec.shape
        assert T % 2 == 0, "frame count must be even (TextAudioSpeakerCollate pads to 2*(Tmax//2+1))"
        I = self.inter_channels
        seg = self.segment_size
        ge = self._ref_enc(spec, lengths)                                        # [B, 1, 512]
        commit = None
        if self.quantizer_trainable:
            quantized, codes, commit = self._quantize_train(ssl, vq_rows, kmeans_idx)
        else:
            with torch.no_grad():                                                # frozen quantizer (models.py:911-921)
                # exact fp32 products: a TF32-rounded (even a 3xTF32) projection flips the argmin of near-tie codewords
                # (measured at the benchmarked shapes: 2, resp. 1, of 1 384 codes); the layer is 1 % of the forward flops
                s = ops.conv_k2s2_fp32(ssl, self.P("ssl_proj.weight"), self.P("ssl_proj.bias"))
                embed = self.P("quantizer.vq.layers.0._codebook.embed")
                codes = ops.vq_nearest(s, embed)                                 # [B, T/2] int64
                quantized = ops.embedding(embed, codes, rep=2)                   # nearest x2 (models.py:924-927)
        # The prior encoder (12 attention layers of small kernels, none of which fills the GPU) only meets the rest of the
        # step again at the KL loss: run it on a side stream so that it overlaps the posterior encoder / flow / generator
        # (forward AND backward: autograd runs each node on its forward stream).  Inside a captured CUDA graph the fork/join
        # becomes two parallel branches.
        side = self._side_stream(spec.device) if SIDE_STREAMS else None
        if side is not None:
            cur = torch.cuda.current_stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                stats_p = self._enc_p(quantized, lengths, text, text_lengths, ge)
            for t in (quantized, ge):
                t.record_stream(side)
            stats_p.record_stream(cur)
        else:
            stats_p = self._enc_p(quantized, lengths, text, text_lengths, ge)
        m_p, logs_p = stats_p[:, :, :I], stats_p[:, :, I:]
        # enc_q, models.py:348-359
        spec_w = ops.widen_to_pitch(spec)      # [B,T,1028]: the 3 pitch columns are zero, enc_q.pre's packed weight is padded alike
        x = ops.linear(spec_w, self.w("enc_q.pre", pad1=spec_w.shape[-1]), self.b("enc_q.pre"), out_len=lengths)
        x = self._wn_stack("enc_q.enc", x, lengths, ge.detach(), 16)
        stats_q = ops.linear(x, self.w("enc_q.proj"), self.b("enc_q.proj"), out_len=lengths)
        if noise is None:
            noise = ops.randn((B, T, I), "enc_q.noise", device=spec.device)
        z = ops.reparam(stats_q, noise, lengths)
        m_q, logs_q = stats_q[:, :, :I], stats_q[:, :, I:]
        # flow, models.py:308-315.  Like the prior encoder it only feeds the KL loss: second side stream, so that its four
        # WaveNet stacks overlap the generator and the discriminators.
        side2 = self._side_stream(spec.device, 1) if SIDE_STREAMS else None
        if side2 is not None:
            cur = torch.cuda.current_stream()
            side2.wait_stream(cur)
            with torch.cuda.stream(side2):
                z_p = self._flow(z, lengths, ge)
            for t in (z, ge):
                t.record_stream(side2)
            z_p.record_stream(cur)
        else:
            z_p = self._flow(z, lengths, ge)
        if ids_slice is None:
            ids_slice = ops.rand_slice_ids(lengths, seg)
        z_slice = ops.slice_rows(z, ids_slice, seg)
        o = self._generator(z_slice, ge)                                         # [B, seg*hop, 1]
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)
        if side2 is not None:
            torch.cuda.current_stream().wait_stream(side2)
        r = dict(y_hat=o, ids_slice=ids_slice, z=z, z_p=z_p, m_p=m_p, logs_p=logs_p, m_q=m_q, logs_q=logs_q,
                 quantized=quantized, codes=codes, ge=ge, lengths=lengths)
        if commit is not None:
            r["kl_ssl"] = commit
        return r

    def forward(self, ssl, y, y_lengths, text, text_lengths, noise=None, ids_slice=None):
        """Reference contract (models.py:904-946): ssl [B,768,T], y = spec [B,1025,T], lengths int64.
        Returns (o, commit_loss, ids_slice, y_mask, y_mask, (z, z_p, m_p, logs_p, m_q, logs_q), quantized) in [B,C,T]."""
        ssl_cl = ops.to_channels_last(ssl)
        spec_cl = ops.to_channels_last(y, pad_to=4)
        ln = y_lengths.to(torch.int32)
        tl = text_lengths.to(torch.int32)
        if noise is not None:
            noise = ops.to_channels_last(noise)
        r = self.forward_cl(ssl_cl, spec_cl, ln, text, tl, noise, ids_slice)
        cf = ops.to_channels_first
        T = y.shape[2]
        y_mask = (torch.arange(T, device=y.device)[None, :] < y_lengths[:, None]).unsqueeze(1).to(y.dtype)
        commit = r.get("kl_ssl", torch.zeros((), device=y.device))     # frozen quantizer: commit_loss == 0
        lat = tuple(cf(r[k]) for k in ("z", "z_p", "m_p", "logs_p", "m_q", "logs_q"))
        return cf(r["y_hat"]), commit, r["ids_slice"], y_mask, y_mask, lat, cf(r["quantized"])


    def _flow_reverse(self, z, lengths, ge):
        """ResidualCouplingBlock(reverse=True), models.py:316-319: Flip, then the mean-only coupling inverted
        (modules.py:459-462: x1 = (x1 - m) * mask), flows 3..0."""
        half = self.inter_channels // 2
        for f in reversed(range(4)):
            p = f"flow.flows.{2 * f}"
            z = ops.flip_channels(z)
            x0, x1 = z[:, :, :half], z[:, :, half:]
            h = ops.linear(x0, self.w(p + ".pre"), self.b(p + ".pre"), out_len=lengths)
            h = self._wn_stack(p + ".enc", h, lengths, ge, 4)
            m = ops.linear(h, self.w(p + ".post"), self.b(p + ".post"), out_len=lengths)
            x1 = ops.add(x1, m, 1.0, -1.0, length=lengths)
            z = torch.cat([x0, x1], dim=-1)
        return z

    @torch.no_grad()
    def decode(self, codes, text, refer, noise_scale=0.5, speed=1, noise=None):
        """Reference contract (models.py:973-1013; the vocoder call of `TTS`, inference/tts.py): codes int64 [1, 1, T]
        (n_q, batch, frames at 25 Hz), text int64 [1, X], refer = reference spectrogram [1, 1025, Tr] or a list of them
        (their style vectors are averaged) -> waveform [1, 1, F * hop] with F = 2T frames, or int(2T / speed) + 1 when
        speed != 1 (linear resampling of the prior encoder output, models.py:246-248).  `noise` [1, 192, F] replaces the
        internal normal draw (tests)."""
        was_training = self.training
        self.eval()
        try:
            dev = codes.device
            ge = self.ref_style(refer)
            B, T = codes.shape[1], codes.shape[2]
            lengths = torch.full((B,), 2 * T, device=dev, dtype=torch.int32)
            text_len = torch.full((B,), text.shape[-1], device=dev, dtype=torch.int32)
            embed = self.P("quantizer.vq.layers.0._codebook.embed")
            quantized = ops.embedding(embed, codes[0].contiguous(), rep=2)       # quantizer.decode + nearest x2
            if speed != 1:
                if B != 1:
                    raise ValueError("SynthesizerTrn.decode: speed != 1 takes one utterance at a time, like the reference")
                stats, lengths = self._enc_p(quantized, lengths, text, text_len, ge, speed)
            else:
                stats = self._enc_p(quantized, lengths, text, text_len, ge)      # [B, F, 2 * 192] = [m_p | logs_p]
            if noise is None:
                noise = ops.randn((B, stats.shape[1], self.inter_channels), "decode.noise", device=dev)
            else:
                noise = ops.to_channels_last(noise.float())
            z_p = ops.reparam(stats, noise * float(noise_scale), lengths)        # m_p + noise * exp(logs_p) * noise_scale
            z = self._flow_reverse(z_p, lengths, ge)
            o = self._generator(ops.rowmask(z, lengths), ge)
            return ops.to_channels_first(o)
        finally:
            self.train(was_training)

    @torch.no_grad()
    def decode_batch(self, codes_list, text_list, ge_rows, noise_scale=0.5, noise=None, noise_keys=None):
        """decode at speed 1 for several rows of different lengths in one pass (tts.run_many): codes_list[b] int64 [T_b] (the
        codes of one bucket, its sentences concatenated), text_list[b] int64 [X_b] (their phones), ge_rows [B, 1, 512] (row b's
        style vector: the mean of _ref_enc over its reference spectrograms, ref_style) -> list of B waveforms [2 T_b * hop].
        The prior encoder, the flow and the generator take per-row lengths; the generator writes zeros past each row's length at
        every rate (_generator), so no row reads a neighbour's padding.  noise: None, or a list of [2 T_b, 192] normal draws
        (tests); without it row b's draws are keyed by noise_keys[b] = (seed, index), so they do not depend on the other rows.
        speed != 1 is not batched: use decode, one sentence at a time."""
        was_training = self.training
        self.eval()
        try:
            B, dev, I = len(codes_list), ge_rows.device, self.inter_channels
            T = [int(c.shape[0]) for c in codes_list]
            Tm, Xm = max(T), max(int(t.shape[0]) for t in text_list)
            codes = torch.zeros((B, Tm), dtype=torch.int64, device=dev)
            text = torch.zeros((B, Xm), dtype=torch.int64, device=dev)
            for b in range(B):
                codes[b, :T[b]] = codes_list[b]
                text[b, :text_list[b].shape[0]] = text_list[b]
            lengths = torch.tensor([2 * t for t in T], dtype=torch.int32).to(dev)
            text_len = torch.tensor([int(t.shape[0]) for t in text_list], dtype=torch.int32).to(dev)
            quantized = ops.embedding(self.P("quantizer.vq.layers.0._codebook.embed"), codes, rep=2)
            stats = self._enc_p(quantized, lengths, text, text_len, ge_rows)
            z = torch.zeros((B, 2 * Tm, I), device=dev, dtype=torch.float32)
            for b in range(B):
                if noise is not None:
                    z[b, :2 * T[b]] = noise[b].to(dev, torch.float32)
                else:
                    seed, k = noise_keys[b]
                    state = torch.tensor([int(seed) & (2 ** 63 - 1), int(k) << 40], dtype=torch.int64, device=dev)
                    z[b, :2 * T[b]] = ops.randn((2 * T[b], I), "decode_batch.noise", device=dev, state=state)
            z_p = ops.reparam(stats, z * float(noise_scale), lengths)
            zf = self._flow_reverse(z_p, lengths, ge_rows)
            o = self._generator(ops.rowmask(zf, lengths), ge_rows, lengths)
            hop = o.shape[1] // (2 * Tm)
            return [o[b, :2 * T[b] * hop, 0] for b in range(B)]
        finally:
            self.train(was_training)

    @torch.no_grad()
    def ref_style(self, refer):
        """decode's style vector: the mean of _ref_enc over the reference spectrograms refer ([1, 1025, Tr] or a list) ->
        [1, 1, 512]"""
        was_training = self.training
        self.eval()
        try:
            refers = refer if isinstance(refer, (list, tuple)) else [refer]
            ges = []
            for r in refers:
                rl = torch.full((r.shape[0],), r.shape[2], device=r.device, dtype=torch.int32)
                ges.append(self._ref_enc(ops.to_channels_last(r.float(), pad_to=4), rl))
            return ges[0] if len(ges) == 1 else torch.stack(ges, 0).mean(0)
        finally:
            self.train(was_training)

    @torch.no_grad()
    def extract_latent(self, x, lengths=None):
        """Reference contract (models.py:1015-1018; the one model call of Normalize.token, normalize.py:203):
        x = HuBERT features [B, 768, T] -> semantic tokens `codes.transpose(0, 1)` = int64 [B, 1, T // 2].
        Same two kernels as the frozen quantizer of the training forward: exact-fp32 stride-2 projection + exact-fp32
        nearest-codeword search (token indices are bit-exact against the reference).  `lengths` (frames per row, optional):
        rows may be zero-padded to a common T; tokens past lengths[b] // 2 are set to 0 and must be ignored by the caller."""
        B, C, T = x.shape
        T2 = T // 2                                              # the stride-2 projection drops an odd last frame
        if T2 == 0:
            return torch.zeros((B, 1, 0), device=x.device, dtype=torch.int64)
        ssl = ops.to_channels_last(x[:, :, :2 * T2].float())
        s = ops.conv_k2s2_fp32(ssl, self.P("ssl_proj.weight"), self.P("ssl_proj.bias"))
        codes = ops.vq_nearest(s, self.P("quantizer.vq.layers.0._codebook.embed"))      # [B, T2]
        if lengths is not None:
            keep = torch.arange(T2, device=x.device)[None, :] < (lengths.to(x.device) // 2)[:, None]
            codes = codes * keep
        return codes.unsqueeze(1)


# ====================================================================================================
# MultiPeriodDiscriminator
# ====================================================================================================
class MultiPeriodDiscriminator(ParamTree):
    """models.py:590-614: one DiscriminatorS (:560-587) + DiscriminatorP for periods 2,3,5,7,11 (:481-557)."""
    S_CFG = [(16, 1, 15, 1, 7, 1), (64, 4, 41, 4, 20, 4), (256, 4, 41, 4, 20, 16), (1024, 4, 41, 4, 20, 64),
             (1024, 4, 41, 4, 20, 256), (1024, 1024, 5, 1, 2, 1)]            # (cout, cin/g, k, stride, pad, groups)
    P_CH = [(32, 1), (128, 32), (512, 128), (1024, 512), (1024, 1024)]

    def __init__(self, use_spectral_norm=False):
        super().__init__()
        assert not use_spectral_norm
        for i, (co, cig, k, s, p, g) in enumerate(self.S_CFG):
            n = f"discriminators.0.convs.{i}"
            self._register(n + ".bias", torch.zeros(co))
            self._register(n + ".weight_g", torch.ones(co, 1, 1))
            self._register(n + ".weight_v", torch.zeros(co, cig, k))
        n = "discriminators.0.conv_post"
        self._register(n + ".bias", torch.zeros(1))
        self._register(n + ".weight_g", torch.ones(1, 1, 1))
        self._register(n + ".weight_v", torch.zeros(1, 1024, 3))
        for d in range(1, 6):
            for i, (co, ci) in enumerate(self.P_CH):
                n = f"discriminators.{d}.convs.{i}"
                self._register(n + ".bias", torch.zeros(co))
                self._register(n + ".weight_g", torch.ones(co, 1, 1, 1))
                self._register(n + ".weight_v", torch.zeros(co, ci, 5, 1))
            n = f"discriminators.{d}.conv_post"
            self._register(n + ".bias", torch.zeros(1))
            self._register(n + ".weight_g", torch.ones(1, 1, 1, 1))
            self._register(n + ".weight_v", torch.zeros(1, 1024, 3, 1))
        self.reset_parameters()

    def reset_parameters(self, seed=4321):
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.endswith("weight_v"):
                    _kaiming_uniform_(p, p[0].numel(), g)
                elif name.endswith(".bias"):
                    _kaiming_uniform_(p, self.P(name[:-4] + "weight_v")[0].numel(), g)
            for name, p in self.named_parameters():
                if name.endswith("weight_g"):
                    v = self.P(name[:-1] + "v")
                    p.copy_(v.flatten(1).norm(dim=1).view(p.shape))

    # 1-channel tensors (the waveform, the logits) are carried with 4 channels (3 of them zero, zero weights) so that
    # every layer -- including its data/weight gradients -- runs on the 16-byte-tiled tensor-core kernels.
    def _disc_s(self, x4):
        fmap = []
        x = x4
        for i, (co, cig, k, s, p, g) in enumerate(self.S_CFG):
            n = f"discriminators.0.convs.{i}"
            x = ops.conv(x, self.w(n, pad1=4 if i == 0 else 0), self.b(n), stride=s, pad=p, groups=g, act=ops.ACT_LRELU,
                         slope=LRELU_SLOPE)
            fmap.append(x)
        n = "discriminators.0.conv_post"
        x = ops.take_channels(ops.conv(x, self.w(n, pad0=4), self.b(n, pad=4), pad=1), 1)
        fmap.append(x)
        return x, fmap

    def _disc_p(self, d, x, period):
        B, T, _ = x.shape
        Tp = (T + period - 1) // period * period
        x = ops.pad_channels(ops.reflect_pad_right(x, Tp), 4)
        fmap = []
        for i, s in enumerate((3, 3, 3, 3, 1)):
            n = f"discriminators.{d}.convs.{i}"
            x = ops.conv(x, self.w(n, pad1=4 if i == 0 else 0), self.b(n), stride=s, pad=2, P=period, act=ops.ACT_LRELU,
                         slope=LRELU_SLOPE)
            fmap.append(x)
        n = f"discriminators.{d}.conv_post"
        x = ops.take_channels(ops.conv(x, self.w(n, pad0=4), self.b(n, pad=4), pad=1, P=period), 1)
        fmap.append(x)
        return x, fmap

    def forward_cl(self, y, y_hat, weights_need_grad=True):
        """y, y_hat [B, T, 1] -> per discriminator (logits [2B, J, 1], fmaps list of [2B, J, C]); rows [:B] are the
        real half, rows [B:] the generated half (one 2B pass instead of the reference's two sequential passes).
        weights_need_grad=False (generator step): D weights are constants, so no D weight gradients are computed --
        the reference computes and then discards them (sovits.py:503,511-520)."""
        self._frozen = not weights_need_grad
        self.begin_pack()
        try:
            x = ops.cat_batch(y, y_hat)
            x4 = ops.pad_channels(x, 4)
            if SIDE_STREAMS and x.is_cuda:
                # the six discriminators are independent chains whose later layers are far too small to fill the GPU: spread
                # them over three streams (parallel branches of the captured graph; the backward follows the same streams)
                cur = torch.cuda.current_stream()
                lanes = [None] + [self._side_stream(x.device, k) for k in range(D_LANES - 1)]
                if D_PRIO and D_LANES == 6:
                    # DiscriminatorS (grouped k = 41 convs, the longest of the six chains) on a high-priority stream
                    lanes = [self._side_stream(x.device, 6, priority=-1), None] + lanes[1:5]
                for st in lanes:
                    if st is not None:
                        st.wait_stream(cur)
                        x.record_stream(st); x4.record_stream(st)
                outs = []
                for d in range(6):
                    st = lanes[d % D_LANES]
                    with torch.cuda.stream(st if st is not None else cur):
                        o = self._disc_s(x4) if d == 0 else self._disc_p(d, x, PERIODS[d - 1])
                    if st is not None:
                        for t in (o[0], *o[1]):
                            t.record_stream(cur)
                    outs.append(o)
                for st in lanes:
                    if st is not None:
                        cur.wait_stream(st)
            else:
                outs = [self._disc_s(x4)]
                for d, period in enumerate(PERIODS, start=1):
                    outs.append(self._disc_p(d, x, period))
        finally:
            self.end_pack()
            self._frozen = False
        return outs

    def forward(self, y, y_hat):
        """Reference contract (models.py:601-614): y, y_hat [B,1,T] -> (y_d_rs, y_d_gs, fmap_rs, fmap_gs)."""
        B = y.shape[0]
        outs = self.forward_cl(y.reshape(B, -1, 1), y_hat.reshape(B, -1, 1))      # [B,1,T] and [B,T,1] share memory
        rs, gs, frs, fgs = [], [], [], []
        for d, (logit, fmap) in enumerate(outs):
            rs.append(logit[:B].reshape(B, -1))
            gs.append(logit[B:].reshape(B, -1))
            fr, fg = [], []
            for f in fmap:
                cf = ops.to_channels_first(f)                     # [2B, C, J]
                if d > 0:
                    p = PERIODS[d - 1]
                    cf = cf.reshape(cf.shape[0], cf.shape[1], -1, p)
                fr.append(cf[:B]); fg.append(cf[B:])
            frs.append(fr); fgs.append(fg)
        return rs, gs, frs, fgs
