"""HuBERT forward for the dataset preparation step (SURVEY section 8 row f3, ssl half).

`Normalize.ssl` (reference src/normalization/normalize.py:131-183) resamples every utterance to 16 kHz and calls
`CNHubert(base_path).model(wav16k.unsqueeze(0))["last_hidden_state"]` (src/easevoice/feature_extractor/cnhubert.py:14-33), i.e.
the `transformers.HubertModel` forward WITHOUT the Wav2Vec2 feature-extractor normalisation, on the CPU, re-instantiating the
model per file.  This module is that forward on the library's kernels, same state_dict keys (transformers 5.x naming, the older
`weight_g` / `weight_v` pair of the positional conv is accepted too), same `[B, L] -> {"last_hidden_state": [B, T, 768]}` contract:

  feature extractor  strided Conv1d stack on the wgmma / mma.sync conv kernels, GroupNorm(512, 512) + GELU in one kernel
                     (`evk_instnorm_cl`), exact-erf GELU (`evk_unary` op 6)
  encoder            grouped k = 128 positional conv (weight-norm folded on the host once), 12 post-LN blocks: three Linear
                     launches for q / k / v, batched attention GEMMs + masked softmax (`ops.attention`), LayerNorm kernels

Inference only (no gradients); fp32 storage, TF32 tensor-core products like the rest of the library.  No CPU fallback.
"""
import json
import os

import torch

from . import ops
from .models import ParamTree

HUBERT_BASE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
                   conv_dim=(512,) * 7, conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2), conv_bias=False,
                   feat_extract_norm="group", do_stable_layer_norm=False, num_conv_pos_embeddings=128,
                   num_conv_pos_embedding_groups=16, layer_norm_eps=1e-5, hidden_act="gelu", feat_extract_activation="gelu")


class HubertModel(ParamTree):
    """transformers.HubertModel (modeling_hubert.py) for the base architecture the reference ships (chinese-hubert-base)."""

    def __init__(self, config=None):
        super().__init__()
        c = dict(HUBERT_BASE, **(config or {}))
        assert c["feat_extract_norm"] == "group" and not c["do_stable_layer_norm"] and not c["conv_bias"], "HuBERT-base layout only"
        assert c["hidden_act"] == "gelu" and c["feat_extract_activation"] == "gelu"
        self.cfg = c
        H, cd = c["hidden_size"], c["conv_dim"]
        for i, k in enumerate(c["conv_kernel"]):
            self._register(f"feature_extractor.conv_layers.{i}.conv.weight", torch.zeros(cd[i], 1 if i == 0 else cd[i - 1], k))
            if i == 0:
                self._register("feature_extractor.conv_layers.0.layer_norm.weight", torch.ones(cd[0]))
                self._register("feature_extractor.conv_layers.0.layer_norm.bias", torch.zeros(cd[0]))
        self._register("feature_projection.layer_norm.weight", torch.ones(cd[-1]))
        self._register("feature_projection.layer_norm.bias", torch.zeros(cd[-1]))
        self._register("feature_projection.projection.weight", torch.zeros(H, cd[-1]))
        self._register("feature_projection.projection.bias", torch.zeros(H))
        K, G = c["num_conv_pos_embeddings"], c["num_conv_pos_embedding_groups"]
        self._register("encoder.pos_conv_embed.conv.bias", torch.zeros(H))
        self._register("encoder.pos_conv_embed.conv.parametrizations.weight.original0", torch.ones(1, 1, K))
        self._register("encoder.pos_conv_embed.conv.parametrizations.weight.original1", torch.zeros(H, H // G, K))
        self._register("encoder.layer_norm.weight", torch.ones(H))
        self._register("encoder.layer_norm.bias", torch.zeros(H))
        for i in range(c["num_hidden_layers"]):
            p = f"encoder.layers.{i}."
            for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
                self._register(p + f"attention.{n}.weight", torch.zeros(H, H))
                self._register(p + f"attention.{n}.bias", torch.zeros(H))
            self._register(p + "layer_norm.weight", torch.ones(H))
            self._register(p + "layer_norm.bias", torch.zeros(H))
            self._register(p + "feed_forward.intermediate_dense.weight", torch.zeros(c["intermediate_size"], H))
            self._register(p + "feed_forward.intermediate_dense.bias", torch.zeros(c["intermediate_size"]))
            self._register(p + "feed_forward.output_dense.weight", torch.zeros(H, c["intermediate_size"]))
            self._register(p + "feed_forward.output_dense.bias", torch.zeros(H))
            self._register(p + "final_layer_norm.weight", torch.ones(H))
            self._register(p + "final_layer_norm.bias", torch.zeros(H))

    # ---- loading ----------------------------------------------------------------------------------------------------------
    def load_state_dict(self, sd, strict=True):
        sd = dict(sd)
        sd.pop("masked_spec_embed", None)                           # training-time mask embedding, unused by the forward
        g, v = "encoder.pos_conv_embed.conv.weight_g", "encoder.pos_conv_embed.conv.weight_v"      # transformers < 4.3x naming
        if g in sd:
            sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"] = sd.pop(g)
            sd["encoder.pos_conv_embed.conv.parametrizations.weight.original1"] = sd.pop(v)
        sd = {(k[len("hubert."):] if k.startswith("hubert.") else k): t.float() for k, t in sd.items()}
        return super().load_state_dict(sd, strict=strict)

    @classmethod
    def from_pretrained(cls, base_path, device="cuda"):
        """`HubertModel.from_pretrained(base_path, local_files_only=True)` for a local directory with config.json and
        pytorch_model.bin (or model.safetensors when the `safetensors` package is importable)."""
        if not os.path.exists(base_path):
            raise FileNotFoundError(base_path)
        cfg = {}
        cj = os.path.join(base_path, "config.json")
        if os.path.exists(cj):
            raw = json.load(open(cj))
            cfg = {k: (tuple(raw[k]) if isinstance(raw[k], list) else raw[k]) for k in HUBERT_BASE if k in raw}
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
    POS_PIECE = 48           # taps per launch of the positional conv (the descriptor holds EVK_MAX_TAPS = 48 tap offsets)

    def _pos_weight(self):
        """weight_norm(dim=2) folded once per parameter version: w[:, :, k] = g[k] * v[:, :, k] / ||v[:, :, k]||_F.
        The k = 128 kernel is packed as ceil(128 / 48) tap pieces (one launch each, chained through the residual input)."""
        g = self.P("encoder.pos_conv_embed.conv.parametrizations.weight.original0")
        v = self.P("encoder.pos_conv_embed.conv.parametrizations.weight.original1")
        key = (int(g._version), int(v._version), str(v.device))
        c = self.__dict__.get("_posw")
        if c is None or c[0] != key:
            w = v * (g / v.norm(p=2, dim=(0, 1), keepdim=True))
            K = w.shape[2]
            pieces = [(a, min(K, a + self.POS_PIECE)) for a in range(0, K, self.POS_PIECE)]
            c = (key, [(a, b, ops.pack_weight(w[:, :, a:b].contiguous(), None, need_pb=False)) for a, b in pieces])
            self.__dict__["_posw"] = c
        return c[1]

    def _pos_conv(self, h):
        """HubertPositionalConvEmbedding (modeling_hubert.py): grouped Conv1d(k = 128, pad = 64) + HubertSamePadLayer (drops the
        last output when k is even) + GELU.  out[t] = sum_q w[q] x[t + q - 64], t < T: every tap piece reads its own window of
        the zero-padded input and adds to the previous piece's output in the epilogue."""
        c = self.cfg
        K, T = c["num_conv_pos_embeddings"], h.shape[1]
        xp = torch.nn.functional.pad(h, (0, 0, K // 2, K // 2 - (1 if K % 2 == 0 else 0)))      # exactly the rows outputs 0..T-1 read
        pos = None
        for a, b, wp in self._pos_weight():
            xin = xp[:, a:a + T + (b - a) - 1].contiguous()
            pos = ops.conv(xin, wp, self.P("encoder.pos_conv_embed.conv.bias") if pos is None else None, pad=0,
                           groups=c["num_conv_pos_embedding_groups"], res=pos)
        return ops.gelu(pos)

    @torch.no_grad()
    def forward(self, input_values):
        """input_values [B, L] float (16 kHz samples, un-normalised as Normalize.ssl passes them) -> {"last_hidden_state": [B, T, H]}.
        All rows are taken at full length (the reference runs one utterance per call)."""
        c = self.cfg
        self._active, self._memo_pack = self.packed_for_inference(), True
        try:
            # channels-last [B, L, 1], widened to 4 zero-padded channels (16-byte rows) like the discriminators' waveform input
            x = ops.pad_channels(input_values.float().unsqueeze(-1).contiguous(), 4)
            for i, (k, s) in enumerate(zip(c["conv_kernel"], c["conv_stride"])):
                w = self.w(f"feature_extractor.conv_layers.{i}.conv", need_pb=False, pad1=4 if i == 0 else 0)
                x = ops.conv(x, w, None, stride=s)
                if i == 0:
                    x = ops.instnorm_cl(x, self.P("feature_extractor.conv_layers.0.layer_norm.weight"),
                                        self.P("feature_extractor.conv_layers.0.layer_norm.bias"), c["layer_norm_eps"], gelu_after=True)
                else:
                    x = ops.gelu(x)
            eps = c["layer_norm_eps"]
            x = ops.layernorm(x, self.P("feature_projection.layer_norm.weight"), self.P("feature_projection.layer_norm.bias"), eps=eps)
            h = ops.linear(x, self.w("feature_projection.projection", need_pb=False), self.b("feature_projection.projection"))
            pos = self._pos_conv(h)
            h = ops.layernorm(h, self.P("encoder.layer_norm.weight"), self.P("encoder.layer_norm.bias"), res=pos, eps=eps)
            H = c["num_attention_heads"]
            scale = (c["hidden_size"] // H) ** -0.5
            for i in range(c["num_hidden_layers"]):
                p = f"encoder.layers.{i}."
                q = ops.linear(h, self.w(p + "attention.q_proj", need_pb=False), self.b(p + "attention.q_proj"))
                k = ops.linear(h, self.w(p + "attention.k_proj", need_pb=False), self.b(p + "attention.k_proj"))
                v = ops.linear(h, self.w(p + "attention.v_proj", need_pb=False), self.b(p + "attention.v_proj"))
                a = ops.attention(q, k, v, heads=H, scale=scale, tag=f"hubert.attn{i}")
                a = ops.linear(a, self.w(p + "attention.out_proj", need_pb=False), self.b(p + "attention.out_proj"))
                h = ops.layernorm(h, self.P(p + "layer_norm.weight"), self.P(p + "layer_norm.bias"), res=a, eps=eps)
                f = ops.gelu(ops.linear(h, self.w(p + "feed_forward.intermediate_dense", need_pb=False),
                                        self.b(p + "feed_forward.intermediate_dense")))
                f = ops.linear(f, self.w(p + "feed_forward.output_dense", need_pb=False), self.b(p + "feed_forward.output_dense"))
                h = ops.layernorm(h, self.P(p + "final_layer_norm.weight"), self.P(p + "final_layer_norm.bias"), res=f, eps=eps)
            return {"last_hidden_state": h}
        finally:
            self._active, self._memo_pack = None, False


class CNHubert(torch.nn.Module):
    """cnhubert.py:14-33: `.model` is the HubertModel; Normalize.ssl calls `.model(wav16k.unsqueeze(0))["last_hidden_state"]`.
    (`forward` of the reference additionally runs Wav2Vec2FeatureExtractor = zero-mean / unit-variance per utterance.)"""

    def __init__(self, base_path, eval=False, device="cuda"):
        super().__init__()
        self.model = HubertModel.from_pretrained(str(base_path), device=device)

    @torch.no_grad()
    def forward(self, x):
        v = x.float()
        if v.dim() == 1:
            v = v.unsqueeze(0)
        v = (v - v.mean(dim=-1, keepdim=True)) / torch.sqrt(v.var(dim=-1, keepdim=True, unbiased=False) + 1e-7)
        return self.model(v.to(next(self.model.parameters()).device))["last_hidden_state"]
