"""UVR5 BS-Roformer vocal separation on the library's kernels: the BSRoformer of lib_v5/vr_network/bs_roformer.py:327-553
(inference) and a batched drop-in for SeparateMDXC.demix_track (uvr5/separate.py:492-574).

Activations stay in one [B, T, bands, dim] layout, B*T*bands rows of `dim` floats.  The time transformer attends over the
T rows of each (b, band) at a stride of `bands` rows, the frequency transformer over the `bands` consecutive rows of each
(b, t); evk_rope_attn_fwd takes both as stride descriptions, so the reference's per-layer 'b t f d -> b f t d' permutes
are never made.  Every RMSNorm is an L2 normalisation (evk_row_l2norm, evk_bs_band_input) whose gamma * sqrt(dim) is folded
into the next Linear's weight columns at load; to_gates is appended to to_qkv as extra output rows.  Linears run on the
TF32 tensor-core GEMM (3xTF32 under evk_set_precise(1)) with GELU, tanh and residual adds in its epilogue.  The complex mask
multiply is fused into the inverse STFT.  Dropout is the identity.
"""
import math

import numpy as np
import torch

from . import lib, ops

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


class BSRoformer:
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
        n_fft = int(stft_n_fft)
        bands = tuple(int(f) for f in freqs_per_bands)
        if dim_head != 64:
            raise ValueError(f"dim_head must be 64, got {dim_head}")
        if linear_transformer_depth != 0:
            raise ValueError("linear_transformer_depth > 0 (LinearAttention) is not supported")
        if num_stems != 1:
            raise ValueError(f"num_stems must be 1, got {num_stems}")
        if n_fft < 256 or n_fft > 4096 or n_fft & (n_fft - 1):
            raise ValueError(f"stft_n_fft must be a power of two in [256, 4096], got {n_fft}")
        if stft_win_length != n_fft:
            raise ValueError(f"stft_win_length ({stft_win_length}) must equal stft_n_fft ({n_fft})")
        if stft_normalized or stft_window_fn is not None:
            raise ValueError("only the default un-normalised Hann STFT is supported")
        if not 0 < stft_hop_length <= n_fft // 2:
            raise ValueError(f"stft_hop_length must be in [1, n_fft // 2], got {stft_hop_length}")
        if len(bands) < 2 or min(bands) < 1 or sum(bands) != n_fft // 2 + 1:
            raise ValueError(f"freqs_per_bands must sum to n_fft // 2 + 1 = {n_fft // 2 + 1}, got {sum(bands)}")
        if dim < 4 or dim % 4 or heads < 1 or depth < 1 or mask_estimator_depth < 1:
            raise ValueError(f"bad sizes: dim {dim} (a multiple of 4), heads {heads}, depth {depth}, "
                             f"mask_estimator_depth {mask_estimator_depth}")
        self.dim, self.depth, self.heads = int(dim), int(depth), int(heads)
        self.stereo, self.S = bool(stereo), 2 if stereo else 1
        self.t_depth, self.f_depth = int(time_transformer_depth), int(freq_transformer_depth)
        self.bands, self.n_fft, self.hop = bands, n_fft, int(stft_hop_length)
        self.mask_depth = int(mask_estimator_depth)
        self.device = torch.device("cpu")
        self.host_w, self.bias = None, None
        self._packed = {}
        self._rope = {}

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _dims_in(self):
        return [2 * f * self.S for f in self.bands]

    def state_dict_shapes(self):
        """-> {key: shape} of the reference's BSRoformer(**config).state_dict() (rotary modules hold no state there)"""
        dim, inner = self.dim, self.heads * 64
        spec = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                for j in range(n):
                    p = f"layers.{i}.{a}.layers.{j}"
                    spec.update({p + ".0.norm.gamma": (dim,), p + ".0.to_qkv.weight": (3 * inner, dim),
                                 p + ".0.to_gates.weight": (self.heads, dim), p + ".0.to_gates.bias": (self.heads,),
                                 p + ".0.to_out.0.weight": (dim, inner), p + ".1.net.0.gamma": (dim,),
                                 p + ".1.net.1.weight": (4 * dim, dim), p + ".1.net.1.bias": (4 * dim,),
                                 p + ".1.net.4.weight": (dim, 4 * dim), p + ".1.net.4.bias": (dim,)})
        spec["final_norm.gamma"] = (dim,)
        for i, d in enumerate(self._dims_in()):
            p = f"band_split.to_features.{i}"
            spec.update({p + ".0.gamma": (d,), p + ".1.weight": (dim, d), p + ".1.bias": (dim,)})
        for i, d in enumerate(self._dims_in()):
            io = [dim] + [4 * dim] * (self.mask_depth - 1) + [2 * d]
            for k in range(self.mask_depth):
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
        missing = [k for k in spec if k not in sd]
        unexpected = [k for k in sd if k not in spec]
        if missing or unexpected:
            raise ValueError(f"state_dict does not match BSRoformer: missing {missing[:5]}{'...' if len(missing) > 5 else ''}, "
                             f"unexpected {unexpected[:5]}{'...' if len(unexpected) > 5 else ''}")
        for k, shape in spec.items():
            v = sd[k]
            if not torch.is_tensor(v) or not v.is_floating_point() or tuple(v.shape) != tuple(shape):
                raise ValueError(f"{k}: expected a float tensor of shape {tuple(shape)}, got "
                                 f"{tuple(v.shape) if torch.is_tensor(v) else type(v).__name__}")
        folded = self._fold({k: sd[k].detach().cpu().to(torch.float32) for k in spec})
        # unpacked weights stay on the host (each precision mode packs its own device copy from them); biases go to the device
        self.host_w = {k[:-2]: v for k, v in folded.items() if k.endswith(".w")}
        self.bias = {k: v.to(self.device) for k, v in folded.items() if k.endswith(".b")}
        self._packed = {}
        return self

    def _fold(self, sd):
        """RMSNorm gamma * sqrt(dim) into the next Linear's columns (in float64), to_gates appended to to_qkv"""
        def fold(w, gamma):
            return (w.double() * (gamma.double() * math.sqrt(gamma.numel()))[None, :]).float()

        D, H = self.heads * 64, self.heads
        ldq = (3 * D + H + 3) // 4 * 4
        out = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                for j in range(n):
                    p = f"layers.{i}.{a}.layers.{j}"
                    g = sd[p + ".0.norm.gamma"]
                    w = torch.zeros(ldq, self.dim)
                    w[:3 * D] = sd[p + ".0.to_qkv.weight"]
                    w[3 * D:3 * D + H] = sd[p + ".0.to_gates.weight"]
                    b = torch.zeros(ldq)
                    b[3 * D:3 * D + H] = sd[p + ".0.to_gates.bias"]
                    out[p + ".qkvg.w"], out[p + ".qkvg.b"] = fold(w, g), b
                    out[p + ".out.w"] = sd[p + ".0.to_out.0.weight"]
                    out[p + ".ff1.w"] = fold(sd[p + ".1.net.1.weight"], sd[p + ".1.net.0.gamma"])
                    out[p + ".ff1.b"] = sd[p + ".1.net.1.bias"]
                    out[p + ".ff2.w"], out[p + ".ff2.b"] = sd[p + ".1.net.4.weight"], sd[p + ".1.net.4.bias"]
        for i in range(len(self.bands)):
            p = f"band_split.to_features.{i}"
            out[f"band.{i}.w"] = fold(sd[p + ".1.weight"], sd[p + ".0.gamma"])
            out[f"band.{i}.b"] = sd[p + ".1.bias"]
            for k in range(self.mask_depth):
                q = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
                w = sd[q + ".weight"]
                out[f"mask.{i}.{k}.w"] = fold(w, sd["final_norm.gamma"]) if k == 0 else w
                out[f"mask.{i}.{k}.b"] = sd[q + ".bias"]
        return out

    def to(self, device):
        self.device = torch.device(device)
        if self.bias is not None:
            self.bias = {k: v.to(self.device) for k, v in self.bias.items()}
        self._packed, self._rope = {}, {}
        return self

    def eval(self):
        """Inference only already (dropout is the identity): returns self, so `SeparateMDXC.separate`'s model.eval() works."""
        return self

    def _weights(self):
        """PackedW operands per precision mode (the packing rounds to TF32 unless evk_set_precise(1) is on)"""
        mode = lib.init().evk_get_precise()
        if mode not in self._packed:
            self._packed[mode] = {k: ops.pack_weight(v.to(self.device), None, need_pb=False) for k, v in self.host_w.items()}
        return self._packed[mode]

    def _rope_table(self, L):
        """[L, 32, 2] (cos, sin) of fp32(p * theta_i), computed in fp32 with accurate cos / sin as rotary_embedding_torch does"""
        if L not in self._rope:
            inv = 1.0 / (ROPE_THETA ** (torch.arange(0, 64, 2).float() / 64))
            ang = torch.arange(L, dtype=torch.float32)[:, None] * inv[None, :]
            self._rope[L] = torch.stack([ang.cos(), ang.sin()], -1).contiguous().to(self.device)
        return self._rope[L]

    @classmethod
    def from_pretrained(cls, path, device="cuda"):
        """The SeparateMDXC model (SHIPPED_CONFIG) with the weights of a reference checkpoint file, on `device`."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(**SHIPPED_CONFIG).to(device).load_state_dict(sd)

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
            ops.row_l2norm(x, out=h)
            wq = W[q + ".qkvg"]
            qkvg = ops.linear_into(h, wq, torch.empty((R, wq.D0), device=x.device), bias=sd[q + ".qkvg.b"])
            a = ops.rope_attn(qkvg, cs, torch.empty((R, D), device=x.device), self.heads, L, *geo)
            del qkvg
            x = ops.linear_into(a, W[q + ".out"], torch.empty_like(x), res=x)
            del a
            ops.row_l2norm(x, out=h)
            f = ops.linear_into(h, W[q + ".ff1"], torch.empty((R, 4 * self.dim), device=x.device), bias=sd[q + ".ff1.b"],
                                act=ops.ACT_GELU)
            x = ops.linear_into(f, W[q + ".ff2"], torch.empty_like(x), bias=sd[q + ".ff2.b"], res=x)
            del f
        return x

    @torch.no_grad()
    def forward(self, raw_audio):
        """raw_audio CUDA [B, S, L] (or [B, L] when mono) -> [B, S, hop * (L // hop)], as the reference's forward"""
        x = self.check_input(raw_audio)
        B, S, L = x.shape
        dev, dim, nb, NB = x.device, self.dim, len(self.bands), self.n_fft // 2 + 1
        W, sd = self._weights(), self.bias
        cplx = ops.stft(x.view(B * S, L), self.n_fft, self.hop)                     # [B*S, T, NB, 2]
        T = cplx.shape[1]
        off = np.concatenate([[0], np.cumsum(self.bands)])
        feat = ops.bs_band_input(cplx, B, S, torch.tensor(off, dtype=torch.int32).to(dev),
                                 torch.empty((B * T, 2 * S * NB), device=dev))
        h = torch.empty((B * T, nb * dim), device=dev)
        for i in range(nb):
            ops.linear_into(feat[:, 2 * S * off[i]:2 * S * off[i + 1]], W[f"band.{i}"], h[:, i * dim:(i + 1) * dim],
                            bias=sd[f"band.{i}.b"])
        del feat
        x = h.view(B * T * nb, dim)
        cs_t, cs_f = self._rope_table(T), self._rope_table(nb)
        for i in range(self.depth):
            x = self._transformer(x, f"layers.{i}.0", self.t_depth, cs_t, T, (B, T * nb, nb, 1, nb))
            x = self._transformer(x, f"layers.{i}.1", self.f_depth, cs_f, nb, (B * T, nb, 1, 0, 1))
        xn = ops.row_l2norm(x).view(B * T, nb * dim)
        del x
        mask = torch.empty((B * T, 2 * S * NB), device=dev)
        for i in range(nb):
            hc = xn[:, i * dim:(i + 1) * dim]
            for k in range(self.mask_depth):
                w = W[f"mask.{i}.{k}"]
                last = k == self.mask_depth - 1
                hc = ops.linear_into(hc, w, torch.empty((B * T, w.D0), device=dev), bias=sd[f"mask.{i}.{k}.b"],
                                     act=ops.ACT_NONE if last else ops.ACT_TANH)
            ops.glu_into(hc, mask[:, 2 * S * off[i]:2 * S * off[i + 1]])
        del xn
        out = ops.istft(cplx, B, S, self.n_fft, self.hop, mask=mask)
        return out.view(B, S, -1)

    __call__ = forward


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
    [S, n]}.  Chunks of CHUNK samples with no overlap; the last is reflect-padded when longer than CHUNK // 2 + 1, else
    zero-padded.  `max_chunks` chunks go through the model per call and the result reaches the host once.  Each chunk's
    output is the model's output, except the samples whose fade weight is 0 under the reference's batches of four, which are
    0 (the reference divides 0 by 0 there and replaces the NaN)."""
    mix = np.asarray(mix.cpu().numpy() if torch.is_tensor(mix) else mix, dtype=np.float32)
    if mix.ndim != 2 or mix.shape[1] < 1:
        raise ValueError(f"mix must be [channels, samples], got {mix.shape}")
    if max_chunks < 1:
        raise ValueError("max_chunks must be >= 1")
    if CHUNK % model.hop:
        raise ValueError(f"the model's hop {model.hop} must divide the chunk length {CHUNK}")
    S, n = mix.shape
    c = CHUNK
    starts, lengths, _ = chunk_plan(n, c)
    tail = mix[:, starts[-1]:]
    if lengths[-1] < c:
        pad = ((0, 0), (0, c - lengths[-1]))
        tail = np.pad(tail, pad, mode="reflect") if lengths[-1] > c // 2 + 1 else np.pad(tail, pad)
    padded = torch.from_numpy(np.ascontiguousarray(np.concatenate([mix[:, :starts[-1]], tail], 1))).to(device)
    nch = len(starts)
    out = torch.empty((S, nch * c), device=device, dtype=torch.float32)
    for j0 in range(0, nch, max_chunks):
        k = min(max_chunks, nch - j0)
        batch = padded[:, j0 * c:(j0 + k) * c].reshape(S, k, c).transpose(0, 1).contiguous()
        out.view(S, nch, c)[:, j0:j0 + k] = model.forward(batch).transpose(0, 1)
    z = zeroed_samples(n, c)
    if len(z):
        out[:, torch.from_numpy(z).to(device)] = 0.0
    return {"vocals": out[:, :n].cpu().numpy()}
