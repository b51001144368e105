"""UVR5 MDX23C separation on the library's kernels: the TFC-TDF v3 U-Net (`TFC_TDF_net` of
lib_v5/vr_network/tfc_tdf_v3.py), inference only, run chunk by chunk through bs_roformer.demix_track.

Activations are channels-last fp32 [B, T, F, C] with the spatial axes (time frame, frequency bin): the reference's layout
after its `transpose(-1, -2)`, which the 1x1 convolutions before and after the U-Net do not notice.  The decoder's
`torch.cat([upscale, skip], 1)` is a buffer per scale: the encoder writes its output into the upper channels, the transposed
conv into the lower ones.  Every conv and Linear is preceded by InstanceNorm + GELU, which run as one pass
(evk_instnorm_plane) into a fresh operand.  Kernels:
  * 3x3, 1x1 and the 2x2 stride-2 downscale: evk_conv2d_fwd; the final 1x1's GELU in its epilogue;
  * the 2x2 stride-2 upscale: evk_convt2x2_fwd, written into the concat buffer;
  * the TDF Linears along the frequency axis: evk_mdx_tdf, the residual `x + tdf(x)` in its epilogue;
  * the 8192-point STFT and iSTFT: evk_stft_fwd / evk_istft, with evk_mdx_front / evk_mdx_back for cac2cws / cws2cac;
  * the shortcut adds, and the last one's `x * first_conv_out`: evk_mdx_add.
Every contraction honours evk_set_precise(1) (3xTF32).

set_compute_type(torch.float16 / torch.bfloat16) runs every evk_conv2d_fwd call on evk_conv2d_fwd_h16 instead (the fp32 input
and the conv weight rounded to 16 bits, fp32 accumulation and epilogue): the 3x3s, the 1x1s, the shortcuts, the 2x2
downscales and final_conv.  The instance norms, GELU, the TDF Linears, the transposed convs, the STFT and the iSTFT stay fp32.
"""
import os
from collections.abc import Mapping

import torch

from . import ops
from .ops import CLView
from .weights import check_state_dict, to_device

# The published 8K-FFT InstVoc HQ configuration, written from memory: no checkpoint or YAML of it was at hand to confirm
# these values.  from_pretrained overrides everything the weights determine.
DEFAULT_CONFIG = {
    "audio": {"chunk_size": 261120, "dim_f": 4096, "dim_t": 256, "hop_length": 1024, "n_fft": 8192, "num_channels": 2,
              "sample_rate": 44100, "min_mean_abs": 0.001},
    "model": {"act": "gelu", "bottleneck_factor": 4, "growth": 128, "norm": "InstanceNorm", "num_blocks_per_scale": 2,
              "num_channels": 128, "num_scales": 5, "num_subbands": 4, "scale": [2, 2]},
    "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": None},
}
EPS = 1e-5


def _get(cfg, path, default=None):
    """cfg.a.b for a mapping or an attribute-style object; default when a part is missing"""
    v = cfg
    for part in path.split("."):
        if isinstance(v, Mapping):
            if part not in v:
                return default
            v = v[part]
        elif hasattr(v, part):
            v = getattr(v, part)
        else:
            return default
    return v


def load_config(config):
    """A mapping, an attribute-style object (SimpleNamespace, ml_collections.ConfigDict) or a path to a YAML file -> the
    object itself (or the parsed YAML)"""
    if isinstance(config, (str, os.PathLike)):
        import yaml
        with open(config) as f:
            return yaml.safe_load(f)
    return config


def _pow2_fft_ok(n):
    return 256 <= n <= 8192 and n & (n - 1) == 0


class MDX23C:
    """MDX23C(config) for inference on CUDA: the reference's TFC_TDF_net(config).  Reads the fields TFC_TDF_net.__init__
    reads (model.*, audio.*, training.instruments / target_instrument) plus audio.chunk_size.  Raises ValueError for what
    the kernels do not take: a norm other than InstanceNorm, an act other than gelu, scale != [2, 2], n_fft not a power of
    two in [256, 8192], hop > n_fft / 2, dim_f > n_fft / 2 + 1, dim_f not divisible by num_subbands * 2^num_scales, and
    chunk_size % hop != 0."""

    def __init__(self, config):
        cfg = load_config(config)
        g = lambda p: _get(cfg, p)   # noqa: E731
        norm, act, scale = g("model.norm"), g("model.act"), g("model.scale")
        if norm != "InstanceNorm":
            raise ValueError(f"model.norm must be InstanceNorm, got {norm!r}")
        if act != "gelu":
            raise ValueError(f"model.act must be gelu, got {act!r}")
        if scale is None or [int(v) for v in scale] != [2, 2]:
            raise ValueError(f"model.scale must be [2, 2], got {scale!r}")
        self.n_fft, self.hop = int(g("audio.n_fft")), int(g("audio.hop_length"))
        self.dim_f, self.S = int(g("audio.dim_f")), int(g("audio.num_channels"))
        self.chunk_size = int(g("audio.chunk_size"))
        self.k, self.n = int(g("model.num_subbands")), int(g("model.num_scales"))
        self.l, self.c0, self.g = int(g("model.num_blocks_per_scale")), int(g("model.num_channels")), int(g("model.growth"))
        self.bn = int(g("model.bottleneck_factor"))
        target, instruments = g("training.target_instrument"), g("training.instruments")
        self.instruments = list(instruments or [])
        self.nt = 1 if target else len(self.instruments)
        if not _pow2_fft_ok(self.n_fft):
            raise ValueError(f"audio.n_fft must be a power of two in [256, 8192], got {self.n_fft}")
        if not 0 < self.hop <= self.n_fft // 2:
            raise ValueError(f"audio.hop_length must be in [1, n_fft // 2], got {self.hop}")
        if not 0 < self.dim_f <= self.n_fft // 2 + 1:
            raise ValueError(f"audio.dim_f must be in [1, n_fft // 2 + 1], got {self.dim_f}")
        if self.k < 1 or self.n < 0 or self.dim_f % (self.k * 2 ** self.n):
            raise ValueError(f"audio.dim_f ({self.dim_f}) must be divisible by num_subbands * 2^num_scales "
                             f"({self.k} * 2^{self.n})")
        if self.chunk_size < 1 or self.chunk_size % self.hop:
            raise ValueError(f"audio.chunk_size ({self.chunk_size}) must be a multiple of hop_length ({self.hop})")
        if self.S < 1 or self.l < 1 or self.c0 < 1 or self.g < 0 or self.bn < 1 or self.nt < 1:
            raise ValueError(f"bad sizes: num_channels {self.S}, num_blocks_per_scale {self.l}, model.num_channels {self.c0}, "
                             f"growth {self.g}, bottleneck_factor {self.bn}, targets {self.nt}")
        f = self.dim_f // self.k
        for _ in range(self.n + 1):
            if f // self.bn < 1:
                raise ValueError(f"bottleneck_factor {self.bn} leaves a TDF Linear with no outputs")
            f //= 2
        self.D = 2 * self.S * self.k
        self.device = torch.device("cpu")
        self.w = None
        self.compute_type = None
        self._h16 = {}

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _tfc_tdf_shapes(self, p, in_c, c, f):
        spec = {}
        for j in range(self.l):
            q = f"{p}.blocks.{j}"
            spec.update({q + ".tfc1.0.weight": (in_c,), q + ".tfc1.0.bias": (in_c,), q + ".tfc1.2.weight": (c, in_c, 3, 3),
                         q + ".tdf.0.weight": (c,), q + ".tdf.0.bias": (c,), q + ".tdf.2.weight": (f // self.bn, f),
                         q + ".tdf.3.weight": (c,), q + ".tdf.3.bias": (c,), q + ".tdf.5.weight": (f, f // self.bn),
                         q + ".tfc2.0.weight": (c,), q + ".tfc2.0.bias": (c,), q + ".tfc2.2.weight": (c, c, 3, 3),
                         q + ".shortcut.weight": (c, in_c, 1, 1)})
            in_c = c
        return spec

    def state_dict_shapes(self):
        """-> {key: shape} of the reference's TFC_TDF_net(config).state_dict(), in its order"""
        c, g, f = self.c0, self.g, self.dim_f // self.k
        spec = {"first_conv.weight": (c, self.D, 1, 1)}
        for i in range(self.n):
            spec.update(self._tfc_tdf_shapes(f"encoder_blocks.{i}.tfc_tdf", c, c, f))
            p = f"encoder_blocks.{i}.downscale.conv"
            spec.update({p + ".0.weight": (c,), p + ".0.bias": (c,), p + ".2.weight": (c + g, c, 2, 2)})
            f //= 2
            c += g
        spec.update(self._tfc_tdf_shapes("bottleneck_block", c, c, f))
        for i in range(self.n):
            p = f"decoder_blocks.{i}.upscale.conv"
            spec.update({p + ".0.weight": (c,), p + ".0.bias": (c,), p + ".2.weight": (c, c - g, 2, 2)})
            f *= 2
            c -= g
            spec.update(self._tfc_tdf_shapes(f"decoder_blocks.{i}.tfc_tdf", 2 * c, c, f))
        spec.update({"final_conv.0.weight": (c, c + self.D, 1, 1), "final_conv.2.weight": (self.nt * self.D, c, 1, 1)})
        return spec

    def load_state_dict(self, sd):
        """Strict load of the reference's state_dict (fp16 or fp32): a missing or unexpected key or a wrong shape raises
        ValueError.  Conv weights are stored [N, kh, kw, C], transposed-conv weights [2, 2, N, C]."""
        spec = self.state_dict_shapes()
        check_state_dict(sd, spec, "MDX23C")
        w = {}
        for k in spec:
            v = sd[k].detach().cpu().to(torch.float32)
            if ".upscale.conv.2." in k:
                v = v.permute(2, 3, 1, 0)
            elif v.dim() == 4:
                v = v.permute(0, 2, 3, 1)
            w[k] = v.contiguous()
        self.host_w = w
        self.w = to_device(w, self.device)
        self._h16 = {}
        return self

    def to(self, device):
        self.device = torch.device(device)
        if self.w is not None:
            self.w = to_device(self.host_w, self.device)
        self._h16 = {}
        return self

    def set_compute_type(self, dtype):
        """None: fp32 activations with TF32 products (the default); torch.float16 or torch.bfloat16: every convolution but
        the transposed ones on evk_conv2d_fwd_h16.  The 16-bit conv weights are packed on first use and kept per compute
        type.  -> self."""
        if dtype is not None and dtype not in ops.H16_TYPES:
            raise ValueError(f"compute type {dtype!r} (None, torch.float16 or torch.bfloat16)")
        self.compute_type = dtype
        return self

    def _h16_weights(self):
        """{key: PackedH16} of every conv weight (4-D, not a transposed conv) for the current 16-bit compute type"""
        key = str(self.compute_type)
        if key not in self._h16:
            self._h16[key] = {k: ops.pack_conv_h16(v, self.compute_type) for k, v in self.w.items()
                              if v.dim() == 4 and ".upscale." not in k}
        return self._h16[key]

    def _conv(self, key, x: CLView, y: CLView, k, stride=1, pad=0, act=ops.C2_NONE):
        """the conv of weight `key` on the compute type's kernel: evk_conv2d_fwd, or evk_conv2d_fwd_h16"""
        if self.compute_type is None:
            ops.conv2d(x, self.w[key], y, k=k, stride=stride, pad=pad, act=act)
        else:
            ops.conv2d_h16(x, self._h16_weights()[key], y, k=k, stride=stride, pad=pad, act=act)

    def eval(self):
        """Inference only already: returns self, so `SeparateMDXC.separate`'s model.eval() works."""
        return self

    @staticmethod
    def infer_config(sd, config=None):
        """The configuration a reference state_dict determines, over `config` (or DEFAULT_CONFIG where config lacks a field):
        model.num_channels, growth, num_scales, num_blocks_per_scale, bottleneck_factor, audio.dim_f (= F * num_subbands
        from the first TDF Linear's F) and the target count.  -> a nested dict."""
        base = load_config(config) if config is not None else {}
        out = {sec: {name: _get(base, f"{sec}.{name}", dv) for name, dv in fields.items()}
               for sec, fields in DEFAULT_CONFIG.items()}
        c0, dim_c = sd["first_conv.weight"].shape[:2]
        n = len({k.split(".")[1] for k in sd if k.startswith("encoder_blocks.")})
        l = len({k.split(".")[4] for k in sd if k.startswith("encoder_blocks.0.tfc_tdf.blocks.")})
        fo, f = sd["encoder_blocks.0.tfc_tdf.blocks.0.tdf.2.weight"].shape
        m = out["model"]
        m.update(num_channels=int(c0), num_scales=n, num_blocks_per_scale=l, bottleneck_factor=int(f // fo))
        if n:
            m["growth"] = int(sd["encoder_blocks.0.downscale.conv.2.weight"].shape[0] - c0)
        k, S = int(m["num_subbands"]), int(out["audio"]["num_channels"])
        if dim_c != 2 * k * S:
            raise ValueError(f"first_conv takes {dim_c} channels; num_subbands {k} and audio.num_channels {S} give {2 * k * S}")
        out["audio"]["dim_f"] = int(f) * k
        nt = int(sd["final_conv.2.weight"].shape[0] // dim_c)
        tr = out["training"]
        ins = list(tr["instruments"] or [])
        if nt > 1:
            tr["target_instrument"] = None
            tr["instruments"] = ins[:nt] + [f"target{i}" for i in range(len(ins), nt)]
        elif not tr["target_instrument"]:
            tr["target_instrument"] = ins[0] if ins else "vocals"
        return out

    @classmethod
    def from_pretrained(cls, path, config=None, device="cuda", compute_type=None):
        """An MDX23C with the weights of a reference checkpoint file, on `device`.  What the weights determine is inferred
        (infer_config); the STFT, chunk and subband settings come from `config` (a mapping, an attribute object or a YAML
        path) or DEFAULT_CONFIG.  compute_type: as set_compute_type."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(cls.infer_config(sd, config)).to(device).load_state_dict(sd).set_compute_type(compute_type)

    # ---- forward -------------------------------------------------------------------------------------------------------
    def _norm(self, key, x: CLView):
        y = torch.empty((x.B, x.H, x.W, x.C), device=self.device)
        return ops.instnorm_plane(x, self.w[key + ".weight"], self.w[key + ".bias"], CLView(y), EPS, True)

    def _tfc_tdf(self, p, x: CLView, out: CLView, mul: CLView = None):
        B, H, W, c = x.B, x.H, x.W, out.C
        new = lambda w, ch: CLView(torch.empty((B, H, w, ch), device=self.device))   # noqa: E731
        for j in range(self.l):
            q = f"{p}.blocks.{j}"
            last = j == self.l - 1
            s = new(W, c)
            self._conv(q + ".shortcut.weight", x, s, k=1)
            t = new(W, c)
            self._conv(q + ".tfc1.2.weight", self._norm(q + ".tfc1.0", x), t, k=3, pad=1)
            u = new(W // self.bn, c)
            ops.mdx_tdf(self._norm(q + ".tdf.0", t), self.w[q + ".tdf.2.weight"], u)
            ops.mdx_tdf(self._norm(q + ".tdf.3", u), self.w[q + ".tdf.5.weight"], t, res=t)
            del u
            t3 = new(W, c)
            self._conv(q + ".tfc2.2.weight", self._norm(q + ".tfc2.0", t), t3, k=3, pad=1)
            del t
            y = out if last else new(W, c)
            ops.mdx_add(t3, s, y, mul if last else None)
            x = y
        return out

    def check_input(self, raw_audio):
        if not torch.is_tensor(raw_audio) or not raw_audio.is_cuda:
            raise ValueError("raw_audio must be a CUDA tensor")
        x = raw_audio
        if x.dim() != 3 or x.shape[1] != self.S or x.shape[0] < 1:
            raise ValueError(f"raw_audio must be [B, {self.S}, L], got {tuple(raw_audio.shape)}")
        L = x.shape[2]
        if L <= self.n_fft // 2:
            raise ValueError(f"raw_audio has {L} samples; the STFT's reflect padding needs more than {self.n_fft // 2}")
        T = 1 + L // self.hop
        if T % (2 ** self.n):
            raise ValueError(f"{L} samples give {T} STFT frames, not divisible by 2^num_scales = {2 ** self.n}")
        if self.w is None:
            raise ValueError("no weights: call load_state_dict first")
        return x.to(torch.float32).contiguous()

    @torch.no_grad()
    def forward(self, raw_audio):
        """raw_audio CUDA [B, S, L] -> [B, n_targets, S, hop * (L // hop)], or [B, S, hop * (L // hop)] for one target"""
        x = self.check_input(raw_audio)
        B, S, L = x.shape
        dev, k, D, c, g = x.device, self.k, self.D, self.c0, self.g
        NB, F = self.n_fft // 2 + 1, self.dim_f // self.k
        cplx = ops.stft(x.view(B * S, L), self.n_fft, self.hop)                    # [B*S, T, NB, 2]
        T = cplx.shape[1]
        fin = torch.empty((B, T, F, D + c), device=dev)                           # final_conv's input: [mix | x * first]
        mix = ops.mdx_front(cplx, B, S, k, F, CLView(fin, 0, D))
        del cplx
        first = CLView(torch.empty((B, T, F, c), device=dev))
        self._conv("first_conv.weight", mix, first, k=1)
        x, h, wd, skips = first, T, F, []
        for i in range(self.n):
            cat = torch.empty((B, h, wd, 2 * c), device=dev)
            enc = self._tfc_tdf(f"encoder_blocks.{i}.tfc_tdf", x, CLView(cat, c, c))
            skips.append(cat)
            p = f"encoder_blocks.{i}.downscale.conv"
            x = CLView(torch.empty((B, h // 2, wd // 2, c + g), device=dev))
            self._conv(p + ".2.weight", self._norm(p + ".0", enc), x, k=2, stride=2)
            c, h, wd = c + g, h // 2, wd // 2
        if self.n == 0:       # the bottleneck is the last block: its output goes straight to final_conv's input
            self._tfc_tdf("bottleneck_block", x, CLView(fin, D, c), first)
        else:
            x = self._tfc_tdf("bottleneck_block", x, CLView(torch.empty((B, h, wd, c), device=dev)))
        for i in range(self.n):
            p = f"decoder_blocks.{i}.upscale.conv"
            cat = skips.pop()
            c, h, wd = c - g, h * 2, wd * 2
            ops.convt2x2(self._norm(p + ".0", x), self.w[p + ".2.weight"], CLView(cat, 0, c))
            last = i == self.n - 1
            out = CLView(fin, D, c) if last else CLView(torch.empty((B, h, wd, c), device=dev))
            x = self._tfc_tdf(f"decoder_blocks.{i}.tfc_tdf", CLView(cat), out, first if last else None)
            del cat
        h1 = CLView(torch.empty((B, T, F, c), device=dev))
        self._conv("final_conv.0.weight", CLView(fin), h1, k=1, act=ops.C2_GELU)
        del fin
        o = CLView(torch.empty((B, T, F, self.nt * D), device=dev))
        self._conv("final_conv.2.weight", h1, o, k=1)
        del h1
        spec = ops.mdx_back(o, self.nt, S, k, NB)
        del o
        out = ops.istft(spec, B * self.nt, S, self.n_fft, self.hop)
        return out.view(B, self.nt, S, -1) if self.nt > 1 else out.view(B, S, -1)

    __call__ = forward
