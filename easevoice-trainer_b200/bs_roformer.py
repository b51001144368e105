"""UVR5 BS-Roformer vocal separation on the library's kernels: the BSRoformer of lib_v5/vr_network/bs_roformer.py:327-553
(inference) and a batched drop-in for SeparateMDXC.demix_track (uvr5/separate.py:492-574).

Activations stay in one [B, T, bands, dim] layout, B*T*bands rows of `dim` floats.  The time transformer attends over the
T rows of each (b, band) at a stride of `bands` rows, the frequency transformer over the `bands` consecutive rows of each
(b, t); evk_rope_attn_fwd takes both as stride descriptions, so the reference's per-layer 'b t f d -> b f t d' permutes
are never made.  Every RMSNorm is an L2 normalisation (evk_row_norm without gamma, evk_band_input) whose gamma * sqrt(dim) is
folded into the next Linear's weight columns at load; to_gates is appended to to_qkv as extra output rows.  Linears run on the
TF32 tensor-core GEMM (3xTF32 under evk_set_precise(1)) with GELU, tanh and residual adds in its epilogue.  The complex mask
multiply is fused into the inverse STFT.  Dropout is the identity.

set_compute_type(torch.float16 / torch.bfloat16) (the reference's is_half) runs every Linear on the 16-bit kernel
(evk_linear_h16: both operands rounded to 16 bits, fp32 accumulation and epilogue) and the attention on
evk_rope_attn_fwd_h16 (rotated q, k, v and the probabilities rounded to 16 bits, fp32 softmax and gate).  The STFT, the band
input, the norms, the GLU, the mask averaging, the inverse STFT, the residual stream and the rotary tables stay fp32.
"""
import math

import numpy as np
import torch

from . import lib, ops
from .weights import check_state_dict, to_device

# SeparateMDXC.get_model_from_config (separate.py:456-490)
SHIPPED_CONFIG = dict(
    attn_dropout=0.1, depth=12, dim=512, dim_freqs_in=1025, dim_head=64, ff_dropout=0.1, flash_attn=True,
    freq_transformer_depth=1,
    freqs_per_bands=(2,) * 24 + (4,) * 12 + (12,) * 8 + (24,) * 8 + (48,) * 8 + (128, 129),
    heads=8, linear_transformer_depth=0, mask_estimator_depth=2, multi_stft_hop_size=147, multi_stft_normalized=False,
    multi_stft_resolution_loss_weight=1.0, multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256), num_stems=1,
    stereo=True, stft_hop_length=441, stft_n_fft=2048, stft_normalized=False, stft_win_length=2048, time_transformer_depth=1,
)
CHUNK = 352800          # demix_track's chunk: 8 s at 44.1 kHz
BATCH = 4               # the reference's chunks per model call (its fade-window rule is per batch of 4)
ROPE_THETA = 10000.0


def check_stft(stft_n_fft, stft_win_length, stft_hop_length, stft_normalized, stft_window_fn):
    """-> n_fft; ValueError for an STFT the kernels do not take (shared by BSRoformer and MelBandRoformer)"""
    n_fft = int(stft_n_fft)
    if n_fft < 256 or n_fft > 4096 or n_fft & (n_fft - 1):
        raise ValueError(f"stft_n_fft must be a power of two in [256, 4096], got {n_fft}")
    if stft_win_length != n_fft:
        raise ValueError(f"stft_win_length ({stft_win_length}) must equal stft_n_fft ({n_fft})")
    if stft_normalized or stft_window_fn is not None:
        raise ValueError("only the default un-normalised Hann STFT is supported")
    if not 0 < stft_hop_length <= n_fft // 2:
        raise ValueError(f"stft_hop_length must be in [1, n_fft // 2], got {stft_hop_length}")
    return n_fft


def check_sizes(dim, heads, depth, mask_estimator_depth):
    if dim < 4 or dim % 4 or heads < 1 or depth < 1 or mask_estimator_depth < 1:
        raise ValueError(f"bad sizes: dim {dim} (a multiple of 4), heads {heads}, depth {depth}, "
                         f"mask_estimator_depth {mask_estimator_depth}")


class AxialRoformer:
    """What BSRoformer and MelBandRoformer share: depth x (time, frequency) Transformers of rotary gated attention and GELU
    feed-forward layers over [B, T, bands, dim] activations, one Linear per band from the band-split operand, one MLP + GLU
    per band to the complex masks, the weight folding and packing, the input checks and the forward pass.  Subclasses
    define the bands: band i holds the bins bins[band_off[i]:band_off[i+1]]; when bands overlap, bin f is held by the slots
    cover[cover_off[f]:cover_off[f+1]] of `bins` and its mask is their average (cover and cover_off None: no overlap).
    match_input_audio_length trims the output to the input's length instead of hop * (L // hop)."""

    def __init__(self, dim, depth, heads, stereo, time_transformer_depth, freq_transformer_depth, n_fft, hop,
                 mask_estimator_depth, mask_linears, bins, band_off, cover=None, cover_off=None,
                 match_input_audio_length=False):
        self.dim, self.depth, self.heads = int(dim), int(depth), int(heads)
        self.stereo, self.S = bool(stereo), 2 if stereo else 1
        self.t_depth, self.f_depth = int(time_transformer_depth), int(freq_transformer_depth)
        self.n_fft, self.hop = n_fft, int(hop)
        self.mask_depth = int(mask_estimator_depth)
        self.mask_linears = int(mask_linears)           # Linears per mask MLP (tanh between them)
        self.chunk_size = CHUNK                         # demix_track's chunk length
        self.bins, self.band_off, self.cover, self.cover_off = bins, band_off, cover, cover_off
        self.match_input_audio_length = bool(match_input_audio_length)
        self.device = torch.device("cpu")
        self.host_w, self.bias = None, None
        self.compute_type = None
        self._packed = {}
        self._rope = {}
        self._tab = None

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _layer_shapes(self, p, n):
        """{key: shape} of the n Attention + FeedForward layers of the Transformer at prefix p"""
        dim, inner = self.dim, self.heads * 64
        spec = {}
        for j in range(n):
            q = f"{p}.layers.{j}"
            spec.update({q + ".0.norm.gamma": (dim,), q + ".0.to_qkv.weight": (3 * inner, dim),
                         q + ".0.to_gates.weight": (self.heads, dim), q + ".0.to_gates.bias": (self.heads,),
                         q + ".0.to_out.0.weight": (dim, inner), q + ".1.net.0.gamma": (dim,),
                         q + ".1.net.1.weight": (4 * dim, dim), q + ".1.net.1.bias": (4 * dim,),
                         q + ".1.net.4.weight": (dim, 4 * dim), q + ".1.net.4.bias": (dim,)})
        return spec

    def _band_shapes(self, dims_in):
        """{key: shape} of band_split and the mask estimator for band-split widths dims_in"""
        dim, spec = self.dim, {}
        for i, d in enumerate(dims_in):
            p = f"band_split.to_features.{i}"
            spec.update({p + ".0.gamma": (d,), p + ".1.weight": (dim, d), p + ".1.bias": (dim,)})
        for i, d in enumerate(dims_in):
            io = [dim] + [4 * dim] * (self.mask_linears - 1) + [2 * d]
            for k in range(self.mask_linears):
                p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
                spec.update({p + ".weight": (io[k + 1], io[k]), p + ".bias": (io[k + 1],)})
        return spec

    def load_state_dict(self, sd):
        """Strict load of the reference's state_dict (fp16 or fp32): a missing or unexpected key or a wrong shape raises
        ValueError.  Checkpoints saved with rotary_embedding_torch also hold each attention's `rotary_embed.freqs`; those are
        accepted when they equal the default frequencies 10000^(-2i / 64) (that is all the kernels compute)."""
        spec = self.state_dict_shapes()
        sd = dict(sd)
        rot = [k for k in sd if k.endswith(".rotary_embed.freqs") and k[: -len("rotary_embed.freqs")] + "to_qkv.weight" in spec]
        ref = 1.0 / (ROPE_THETA ** (torch.arange(0, 64, 2).float() / 64))
        for k in rot:
            v = sd.pop(k)
            ok = torch.is_tensor(v) and v.is_floating_point() and tuple(v.shape) == (32,)
            # the defaults as stored in the checkpoint's dtype (fp16 checkpoints hold them rounded to half precision)
            if not ok or not torch.allclose(v.float().cpu(), ref, rtol=max(torch.finfo(v.dtype).eps, 1e-5), atol=0):
                raise ValueError(f"{k}: only the default rotary frequencies (theta 10000) are supported")
        check_state_dict(sd, spec, type(self).__name__)
        folded = self._fold({k: sd[k].detach().cpu().to(torch.float32) for k in spec})
        # unpacked weights stay on the host (each precision mode packs its own device copy from them); biases (and any
        # other vectors the forward reads) go to the device
        self.host_w = {k[:-2]: v for k, v in folded.items() if k.endswith(".w")}
        self.bias = to_device({k: v for k, v in folded.items() if not k.endswith(".w")}, self.device)
        self._packed = {}
        return self

    @staticmethod
    def _fold_gamma(w, gamma):
        """RMSNorm gamma * sqrt(dim) into the next Linear's columns (in float64)"""
        return (w.double() * (gamma.double() * math.sqrt(gamma.numel()))[None, :]).float()

    def _fold_layers(self, sd, p, n, out):
        """the n layers of the Transformer at prefix p: norm gammas folded, to_gates appended to to_qkv"""
        fold = self._fold_gamma
        D, H = self.heads * 64, self.heads
        ldq = (3 * D + H + 3) // 4 * 4
        for j in range(n):
            q = f"{p}.layers.{j}"
            g = sd[q + ".0.norm.gamma"]
            w = torch.zeros(ldq, self.dim)
            w[:3 * D] = sd[q + ".0.to_qkv.weight"]
            w[3 * D:3 * D + H] = sd[q + ".0.to_gates.weight"]
            b = torch.zeros(ldq)
            b[3 * D:3 * D + H] = sd[q + ".0.to_gates.bias"]
            out[q + ".qkvg.w"], out[q + ".qkvg.b"] = fold(w, g), b
            out[q + ".out.w"] = sd[q + ".0.to_out.0.weight"]
            out[q + ".ff1.w"] = fold(sd[q + ".1.net.1.weight"], sd[q + ".1.net.0.gamma"])
            out[q + ".ff1.b"] = sd[q + ".1.net.1.bias"]
            out[q + ".ff2.w"], out[q + ".ff2.b"] = sd[q + ".1.net.4.weight"], sd[q + ".1.net.4.bias"]

    def _fold_bands(self, sd, nb, mask_gamma, out):
        """band_split (its RMSNorm gammas folded) and the mask MLPs (mask_gamma, the norm before them, folded into layer 0)"""
        fold = self._fold_gamma
        for i in range(nb):
            p = f"band_split.to_features.{i}"
            out[f"band.{i}.w"] = fold(sd[p + ".1.weight"], sd[p + ".0.gamma"])
            out[f"band.{i}.b"] = sd[p + ".1.bias"]
            for k in range(self.mask_linears):
                q = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
                w = sd[q + ".weight"]
                out[f"mask.{i}.{k}.w"] = fold(w, mask_gamma) if k == 0 else w
                out[f"mask.{i}.{k}.b"] = sd[q + ".bias"]

    def to(self, device):
        self.device = torch.device(device)
        if self.bias is not None:
            self.bias = to_device(self.bias, self.device)
        self._packed, self._rope, self._tab = {}, {}, None
        return self

    def eval(self):
        """Inference only already (dropout is the identity): returns self, so `SeparateMDXC.separate`'s model.eval() works."""
        return self

    def set_compute_type(self, dtype):
        """None: fp32 activations with TF32 products (the default); torch.float16 or torch.bfloat16: every Linear and the
        attention on the 16-bit kernels.  The weights are packed for the compute type on the next forward.  -> self."""
        if dtype is not None and dtype not in ops.H16_TYPES:
            raise ValueError(f"compute type {dtype!r} (None, torch.float16 or torch.bfloat16)")
        self.compute_type = dtype
        return self

    def _weights_key(self):
        """(precise mode, compute type): the TF32 packs depend on evk_set_precise, the 16-bit ones on the dtype only"""
        return (lib.init().evk_get_precise() if self.compute_type is None else None, str(self.compute_type))

    def _weights(self):
        """The Linears' packed weights for _weights_key(): PackedW (rounded to TF32 unless evk_set_precise(1) is on) when the
        compute type is None, else only PackedH16 of the compute type"""
        key = self._weights_key()
        if key not in self._packed:
            h16 = self.compute_type
            pk = (lambda w: ops.pack_weight(w, None, need_pb=False)) if h16 is None else (lambda w: ops.pack_weight_h16(w, h16))
            self._packed[key] = {k: pk(v.to(self.device)) for k, v in self.host_w.items()}
        return self._packed[key]

    def _linear(self, x, w, out, bias=None, act=ops.ACT_NONE, res=None):
        """out = act(x W^T + bias + res) on the compute type's kernel: the TF32 GEMM, or evk_linear_h16"""
        if self.compute_type is None:
            return ops.linear_into(x, w, out, bias=bias, act=act, res=res)
        return ops.linear_h16(x, w, bias=bias, act=act, res=res, out=out)

    def _rope_table(self, L):
        """[L, 32, 2] (cos, sin) of fp32(p * theta_i), computed in fp32 with accurate cos / sin as rotary_embedding_torch does"""
        if L not in self._rope:
            inv = 1.0 / (ROPE_THETA ** (torch.arange(0, 64, 2).float() / 64))
            ang = torch.arange(L, dtype=torch.float32)[:, None] * inv[None, :]
            self._rope[L] = torch.stack([ang.cos(), ang.sin()], -1).contiguous().to(self.device)
        return self._rope[L]

    def _tables(self):
        """the band tables as device int32 tensors (bins, band_off, cover, cover_off), None where a table is None"""
        if self._tab is None:
            self._tab = [None if t is None else torch.from_numpy(t).to(self.device)
                         for t in (self.bins, self.band_off, self.cover, self.cover_off)]
        return self._tab

    # ---- forward -------------------------------------------------------------------------------------------------------
    def check_input(self, raw_audio):
        """-> [B, S, L] fp32 contiguous; ValueError for a non-CUDA tensor, the wrong channel count or L <= n_fft // 2"""
        if not torch.is_tensor(raw_audio) or not raw_audio.is_cuda:
            raise ValueError("raw_audio must be a CUDA tensor")
        x = raw_audio
        if x.dim() == 2:
            x = x[:, None]
        if x.dim() != 3 or x.shape[1] != self.S or x.shape[0] < 1:
            raise ValueError(f"raw_audio must be [B, {self.S}, L]{' or [B, L]' if self.S == 1 else ''} "
                             f"(stereo={self.stereo}), got {tuple(raw_audio.shape)}")
        if x.shape[2] <= self.n_fft // 2:
            raise ValueError(f"raw_audio has {x.shape[2]} samples; the STFT's reflect padding needs more than {self.n_fft // 2}")
        if self.bias is None:
            raise ValueError("no weights: call load_state_dict first")
        return x.to(torch.float32).contiguous()

    def _transformer(self, x, p, depth, cs, L, geo):
        D = self.heads * 64
        R = x.shape[0]
        W, sd = self._weights(), self.bias
        h = torch.empty_like(x)
        for j in range(depth):
            q = f"{p}.layers.{j}"
            ops.row_norm(x, out=h)
            b = sd[q + ".qkvg.b"]
            qkvg = self._linear(h, W[q + ".qkvg"], torch.empty((R, b.numel()), device=x.device), bias=b)
            a = torch.empty((R, D), device=x.device)
            if self.compute_type is None:
                ops.rope_attn(qkvg, cs, a, self.heads, L, *geo)
            else:
                ops.rope_attn_h16(qkvg, cs, a, self.heads, L, *geo, self.compute_type)
            del qkvg
            x = self._linear(a, W[q + ".out"], torch.empty_like(x), res=x)
            del a
            ops.row_norm(x, out=h)
            f = self._linear(h, W[q + ".ff1"], torch.empty((R, 4 * self.dim), device=x.device), bias=sd[q + ".ff1.b"],
                             act=ops.ACT_GELU)
            x = self._linear(f, W[q + ".ff2"], torch.empty_like(x), bias=sd[q + ".ff2.b"], res=x)
            del f
        return x

    def _band_split(self, feat, off, rows):
        """band i's Linear on the columns [2 S off[i], 2 S off[i+1]) of the band-split operand -> [rows * bands, dim]"""
        W, sd, S, dim, nb = self._weights(), self.bias, self.S, self.dim, len(off) - 1
        h = torch.empty((rows, nb * dim), device=feat.device)
        for i in range(nb):
            self._linear(feat[:, 2 * S * off[i]:2 * S * off[i + 1]], W[f"band.{i}"], h[:, i * dim:(i + 1) * dim],
                         bias=sd[f"band.{i}.b"])
        return h.view(rows * nb, dim)

    def _mask_estimator(self, xn, off, out):
        """band i's MLP and GLU on its dim columns of xn [rows, bands * dim] -> the columns [2 S off[i], 2 S off[i+1]) of out"""
        W, sd, S, dim, rows = self._weights(), self.bias, self.S, self.dim, xn.shape[0]
        for i in range(len(off) - 1):
            hc = xn[:, i * dim:(i + 1) * dim]
            for k in range(self.mask_linears):
                b = sd[f"mask.{i}.{k}.b"]
                last = k == self.mask_linears - 1
                hc = self._linear(hc, W[f"mask.{i}.{k}"], torch.empty((rows, b.numel()), device=xn.device), bias=b,
                                  act=ops.ACT_NONE if last else ops.ACT_TANH)
            ops.glu_into(hc, out[:, 2 * S * off[i]:2 * S * off[i + 1]])
        return out

    @torch.no_grad()
    def forward(self, raw_audio):
        """raw_audio CUDA [B, S, L] (or [B, L] when mono) -> [B, S, hop * (L // hop)], or [B, S, L] with
        match_input_audio_length, as the reference's forward"""
        x = self.check_input(raw_audio)
        B, S, L = x.shape
        dev, dim, nb, NB, n_slots = x.device, self.dim, len(self.band_off) - 1, self.n_fft // 2 + 1, len(self.bins)
        bins, band_off, cover, cover_off = self._tables()
        cplx = ops.stft(x.view(B * S, L), self.n_fft, self.hop)                     # [B*S, T, NB, 2]
        T = cplx.shape[1]
        feat = ops.band_input(cplx, B, S, band_off, bins, torch.empty((B * T, 2 * S * n_slots), device=dev))
        x = self._band_split(feat, self.band_off, B * T)
        del feat
        cs_t, cs_f = self._rope_table(T), self._rope_table(nb)
        for i in range(self.depth):
            for a, n, cs, Lq, geo in ((0, self.t_depth, cs_t, T, (B, T * nb, nb, 1, nb)),
                                      (1, self.f_depth, cs_f, nb, (B * T, nb, 1, 0, 1))):
                p = f"layers.{i}.{a}"
                x = self._transformer(x, p, n, cs, Lq, geo)
                if p + ".norm.g" in self.bias:                               # a Transformer's own output RMSNorm
                    ops.row_norm(x, self.bias[p + ".norm.g"], out=x)
        xn = ops.row_norm(x).view(B * T, nb * dim)                   # the last norm; its gamma is folded into the mask MLPs
        del x
        # without overlapping bands the GLU writes straight into the mask layout the inverse STFT reads
        mask = self._mask_estimator(xn, self.band_off, torch.empty((B * T, 2 * S * n_slots), device=dev))
        del xn
        if cover is not None:
            mask = ops.melband_mask_avg(mask, S, cover_off, cover, torch.empty((B * T, 2 * S * NB), device=dev))
        out = ops.istft(cplx, B, S, self.n_fft, self.hop, mask=mask, length=L if self.match_input_audio_length else None)
        return out.view(B, S, -1)

    __call__ = forward


class BSRoformer(AxialRoformer):
    """BSRoformer(**config) for inference on CUDA.  Takes the reference's keyword arguments; the training-only ones
    (`*_dropout`, `multi_stft_*`, `flash_attn`) are accepted and ignored.  Raises ValueError for what the kernels do not
    take: dim_head != 64, linear_transformer_depth != 0, num_stems != 1, stft_n_fft not a power of two in [256, 4096],
    stft_win_length != stft_n_fft, stft_normalized, a custom stft_window_fn, a hop above n_fft / 2, and bands that do not
    sum to n_fft // 2 + 1."""

    def __init__(self, dim, *, depth, stereo=False, num_stems=1, time_transformer_depth=2, freq_transformer_depth=2,
                 linear_transformer_depth=0, freqs_per_bands=SHIPPED_CONFIG["freqs_per_bands"], dim_head=64, heads=8,
                 dim_freqs_in=1025, stft_n_fft=2048, stft_hop_length=512, stft_win_length=2048, stft_normalized=False,
                 stft_window_fn=None, mask_estimator_depth=2, attn_dropout=0.0, ff_dropout=0.0, flash_attn=True,
                 multi_stft_resolution_loss_weight=1.0, multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256),
                 multi_stft_hop_size=147, multi_stft_normalized=False, multi_stft_window_fn=None):
        bands = tuple(int(f) for f in freqs_per_bands)
        if dim_head != 64:
            raise ValueError(f"dim_head must be 64, got {dim_head}")
        if linear_transformer_depth != 0:
            raise ValueError("linear_transformer_depth > 0 (LinearAttention) is not supported")
        if num_stems != 1:
            raise ValueError(f"num_stems must be 1, got {num_stems}")
        n_fft = check_stft(stft_n_fft, stft_win_length, stft_hop_length, stft_normalized, stft_window_fn)
        if len(bands) < 2 or min(bands) < 1 or sum(bands) != n_fft // 2 + 1:
            raise ValueError(f"freqs_per_bands must sum to n_fft // 2 + 1 = {n_fft // 2 + 1}, got {sum(bands)}")
        check_sizes(dim, heads, depth, mask_estimator_depth)
        super().__init__(dim, depth, heads, stereo, time_transformer_depth, freq_transformer_depth, n_fft, stft_hop_length,
                         mask_estimator_depth, mask_estimator_depth, np.arange(n_fft // 2 + 1, dtype=np.int32),
                         np.concatenate([[0], np.cumsum(bands)]).astype(np.int32))
        self.bands = bands

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _dims_in(self):
        return [2 * f * self.S for f in self.bands]

    def state_dict_shapes(self):
        """-> {key: shape} of the reference's BSRoformer(**config).state_dict() (rotary modules hold no state there)"""
        spec = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                spec.update(self._layer_shapes(f"layers.{i}.{a}", n))
        spec["final_norm.gamma"] = (self.dim,)
        spec.update(self._band_shapes(self._dims_in()))
        return spec

    def _fold(self, sd):
        """RMSNorm gamma * sqrt(dim) into the next Linear's columns (in float64), to_gates appended to to_qkv"""
        out = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                self._fold_layers(sd, f"layers.{i}.{a}", n, out)
        self._fold_bands(sd, len(self.bands), sd["final_norm.gamma"], out)
        return out

    @classmethod
    def from_pretrained(cls, path, device="cuda", compute_type=None):
        """The SeparateMDXC model (SHIPPED_CONFIG) with the weights of a reference checkpoint file, on `device`.
        compute_type: as set_compute_type."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(**SHIPPED_CONFIG).to(device).load_state_dict(sd).set_compute_type(compute_type)


def chunk_plan(n, c=CHUNK, batch=BATCH):
    """The reference's chunking of an n-sample mix: -> (starts, lengths, window kind per chunk) where the kind is the
    window of the chunk's batch of `batch` (0 start, 1 middle, 2 finish), chosen from the batch's last chunk."""
    starts = list(range(0, n, c))
    lengths = [min(c, n - s) for s in starts]
    kinds = []
    for j in range(len(starts)):
        last = min((j // batch) * batch + batch - 1, len(starts) - 1)
        kinds.append(0 if last == 0 else 2 if last == len(starts) - 1 else 1)
    return starts, lengths, kinds


def zeroed_samples(n, c=CHUNK, batch=BATCH):
    """Sample indices whose fade weight is 0 in the reference's demix_track (0 / 0, then nan_to_num -> 0)"""
    out = []
    for s, l, kind in zip(*chunk_plan(n, c, batch)):
        if kind in (1, 2):
            out.append(s)                            # fade-in starts at 0
        if kind in (0, 1) and l == c:
            out.append(s + c - 1)                    # fade-out ends at 0
    return np.array(sorted(out), dtype=np.int64)


@torch.no_grad()
def demix_track(model, mix, device="cuda", max_chunks=4):
    """SeparateMDXC.demix_track(model, mix, device) on the device: mix [S, n] (torch or numpy, fp32) -> {"vocals": np.ndarray
    [S, n]}, or for a model with several targets {"vocals": target 0, "other": target 1} (the reference's zip over the
    target axis of its estimate).  Chunks of model.chunk_size samples (CHUNK for the roformers) with no overlap; the last is
    reflect-padded when longer than half a chunk + 1, else zero-padded.  `max_chunks` chunks go through the model per call
    and the result reaches the host once.  Each chunk's output is the model's output, except the samples whose fade weight
    is 0 under the reference's batches of four, which are 0 (the reference divides 0 by 0 there and replaces the NaN)."""
    mix = np.asarray(mix.cpu().numpy() if torch.is_tensor(mix) else mix, dtype=np.float32)
    if mix.ndim != 2 or mix.shape[1] < 1:
        raise ValueError(f"mix must be [channels, samples], got {mix.shape}")
    if max_chunks < 1:
        raise ValueError("max_chunks must be >= 1")
    c = int(model.chunk_size)
    if c % model.hop:
        raise ValueError(f"the model's hop {model.hop} must divide the chunk length {c}")
    S, n = mix.shape
    starts, lengths, _ = chunk_plan(n, c)
    tail = mix[:, starts[-1]:]
    if lengths[-1] < c:
        pad = ((0, 0), (0, c - lengths[-1]))
        tail = np.pad(tail, pad, mode="reflect") if lengths[-1] > c // 2 + 1 else np.pad(tail, pad)
    padded = torch.from_numpy(np.ascontiguousarray(np.concatenate([mix[:, :starts[-1]], tail], 1))).to(device)
    nch = len(starts)
    out = None
    for j0 in range(0, nch, max_chunks):
        k = min(max_chunks, nch - j0)
        batch = padded[:, j0 * c:(j0 + k) * c].reshape(S, k, c).transpose(0, 1).contiguous()
        y = model.forward(batch)
        y = y.view(k, -1, S, c)                                     # [chunks, targets, S, c]
        if out is None:
            out = torch.empty((y.shape[1], S, nch * c), device=device, dtype=torch.float32)
        out.view(-1, S, nch, c)[:, :, j0:j0 + k] = y.permute(1, 2, 0, 3)
    z = zeroed_samples(n, c)
    if len(z):
        out[..., torch.from_numpy(z).to(device)] = 0.0
    est = out[..., :n].cpu().numpy()
    return {k: v for k, v in zip(["vocals", "other"], est)}
