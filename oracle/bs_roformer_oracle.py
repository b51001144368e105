"""CPU restatement of the UVR5 BS-Roformer separator: BSRoformer.forward in eval mode (lib_v5/vr_network/bs_roformer.py:327-553,
attend.py) and SeparateMDXC.demix_track (uvr5/separate.py:492-574), in stock torch fp32 with seeded weights.

Key names are the reference's state_dict names (`layers.0.0.layers.0.0.to_qkv.weight`, ...).  Dropout is the identity.
`RotaryEmbedding` is a functional stand-in for rotary_embedding_torch.RotaryEmbedding written from that library's documented
defaults (theta 10000, all dims rotated, interleaved pairs, fp32 angles); it is not taken from the library.
oracle/pin_bs_roformer.py checks this file against the unmodified reference."""
import numpy as np
import torch
import torch.nn.functional as F

SHIPPED = dict(
    attn_dropout=0.1, depth=12, dim=512, dim_freqs_in=1025, dim_head=64, ff_dropout=0.1, flash_attn=True,
    freq_transformer_depth=1,
    freqs_per_bands=(2,) * 24 + (4,) * 12 + (12,) * 8 + (24,) * 8 + (48,) * 8 + (128, 129),
    heads=8, linear_transformer_depth=0, mask_estimator_depth=2, multi_stft_hop_size=147, multi_stft_normalized=False,
    multi_stft_resolution_loss_weight=1.0, multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256), num_stems=1,
    stereo=True, stft_hop_length=441, stft_n_fft=2048, stft_normalized=False, stft_win_length=2048, time_transformer_depth=1,
)
CHUNK = 352800                       # demix_track's c: 8 s at 44.1 kHz


def rotary_inv_freq(dim=64, theta=10000.0):
    """theta_i = 1 / theta^(2i / dim), fp32 (rotary_embedding_torch's default `freqs` of length dim / 2)"""
    return 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))


def rotary_cos_sin(L, dim=64):
    """-> (cos, sin) [L, dim / 2] fp32: angle = fp32(p * theta_i) for positions p = 0 .. L-1"""
    ang = torch.arange(L, dtype=torch.float32)[:, None] * rotary_inv_freq(dim)[None, :]
    return ang.cos(), ang.sin()


class RotaryEmbedding:
    """rotary_embedding_torch.RotaryEmbedding(dim) with its defaults, as BSRoformer uses it: rotate_queries_or_keys(t) rotates
    t [..., n, dim] at positions 0 .. n-1 along the second-to-last axis, pairs (2i, 2i+1) interleaved:
        out[2i] = x[2i] cos - x[2i+1] sin,   out[2i+1] = x[2i+1] cos + x[2i] sin,   angle = p * 10000^(-2i / dim)."""

    def __init__(self, dim, **_):
        self.dim = dim

    def rotate_queries_or_keys(self, t, seq_dim=-2):
        assert seq_dim == -2 and t.shape[-1] == self.dim
        cos, sin = rotary_cos_sin(t.shape[-2], self.dim)
        cos = cos.repeat_interleave(2, -1).to(t.device, t.dtype)
        sin = sin.repeat_interleave(2, -1).to(t.device, t.dtype)
        x = t.unflatten(-1, (-1, 2))
        rot = torch.stack((-x[..., 1], x[..., 0]), -1).flatten(-2)
        return t * cos + rot * sin


def _audio_channels(cfg):
    return 2 if cfg.get("stereo", False) else 1


def param_spec(cfg):
    """-> {state_dict key: shape} of BSRoformer(**cfg) (linear_transformer_depth 0, one stem), in the reference's key order."""
    dim, heads, dh = cfg["dim"], cfg.get("heads", 8), cfg.get("dim_head", 64)
    inner, S = heads * dh, _audio_channels(cfg)
    spec = {}
    for i in range(cfg["depth"]):
        for a, n in ((0, cfg.get("time_transformer_depth", 2)), (1, cfg.get("freq_transformer_depth", 2))):
            for j in range(n):
                p = f"layers.{i}.{a}.layers.{j}"
                spec[p + ".0.norm.gamma"] = (dim,)
                spec[p + ".0.to_qkv.weight"] = (3 * inner, dim)
                spec[p + ".0.to_gates.weight"] = (heads, dim)
                spec[p + ".0.to_gates.bias"] = (heads,)
                spec[p + ".0.to_out.0.weight"] = (dim, inner)
                spec[p + ".1.net.0.gamma"] = (dim,)
                spec[p + ".1.net.1.weight"] = (4 * dim, dim)
                spec[p + ".1.net.1.bias"] = (4 * dim,)
                spec[p + ".1.net.4.weight"] = (dim, 4 * dim)
                spec[p + ".1.net.4.bias"] = (dim,)
    spec["final_norm.gamma"] = (dim,)
    dims = [2 * f * S for f in cfg["freqs_per_bands"]]
    for i, d in enumerate(dims):
        spec[f"band_split.to_features.{i}.0.gamma"] = (d,)
        spec[f"band_split.to_features.{i}.1.weight"] = (dim, d)
        spec[f"band_split.to_features.{i}.1.bias"] = (dim,)
    depth, hid = cfg.get("mask_estimator_depth", 2), 4 * dim
    for i, d in enumerate(dims):
        io = [dim] + [hid] * (depth - 1) + [2 * d]
        for k in range(depth):
            p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
            spec[p + ".weight"] = (io[k + 1], io[k])
            spec[p + ".bias"] = (io[k + 1],)
    return spec


def init_params(spec, seed):
    """Seeded weights: Linear weights N(0, 1 / fan_in), biases N(0, 0.1^2), RMSNorm gammas in [0.5, 1.5]."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for k, shape in spec.items():
        if k.endswith("gamma"):
            P[k] = 0.5 + torch.rand(shape, generator=g)
        elif k.endswith("bias"):
            P[k] = 0.1 * torch.randn(shape, generator=g)
        else:
            P[k] = torch.randn(shape, generator=g) / shape[1] ** 0.5
    return P


def make_audio(seed, shape):
    """Seeded test audio: noise plus two tones, peak about 0.5."""
    g = torch.Generator().manual_seed(seed)
    n = shape[-1]
    t = torch.arange(n, dtype=torch.float64) / 44100.0
    tone = 0.2 * torch.sin(2 * np.pi * 220.0 * t) + 0.1 * torch.sin(2 * np.pi * 3150.0 * t)
    return (0.15 * torch.randn(shape, generator=g, dtype=torch.float64) + tone).float()


def _rms(x, gamma):
    return F.normalize(x, dim=-1) * x.shape[-1] ** 0.5 * gamma


def _transformer(P, p, x, depth, heads, rope):
    for j in range(depth):
        q = f"{p}.layers.{j}"
        h = _rms(x, P[q + ".0.norm.gamma"])
        qkv = F.linear(h, P[q + ".0.to_qkv.weight"])
        n, L = x.shape[0], x.shape[1]
        qq, kk, vv = qkv.reshape(n, L, 3, heads, -1).permute(2, 0, 3, 1, 4)
        qq, kk = rope.rotate_queries_or_keys(qq), rope.rotate_queries_or_keys(kk)
        o = F.scaled_dot_product_attention(qq, kk, vv)
        gates = F.linear(h, P[q + ".0.to_gates.weight"], P[q + ".0.to_gates.bias"])
        o = o * gates.permute(0, 2, 1)[..., None].sigmoid()
        x = F.linear(o.permute(0, 2, 1, 3).reshape(n, L, -1), P[q + ".0.to_out.0.weight"]) + x
        h = _rms(x, P[q + ".1.net.0.gamma"])
        h = F.gelu(F.linear(h, P[q + ".1.net.1.weight"], P[q + ".1.net.1.bias"]))
        x = F.linear(h, P[q + ".1.net.4.weight"], P[q + ".1.net.4.bias"]) + x
    return x


@torch.no_grad()
def forward(P, cfg, raw):
    """BSRoformer(**cfg).forward(raw) in eval mode: raw [B, S, L] (or [B, L] mono) fp32 -> [B, S, hop * (L // hop)]"""
    if raw.dim() == 2:
        raw = raw[:, None]
    B, S, L = raw.shape
    n_fft, hop = cfg["stft_n_fft"], cfg["stft_hop_length"]
    bands, heads, dim = cfg["freqs_per_bands"], cfg.get("heads", 8), cfg["dim"]
    win = torch.hann_window(n_fft, device=raw.device)                 # fp32 whatever the input dtype, as the reference's
    X = torch.view_as_real(torch.stft(raw.reshape(B * S, L), n_fft, hop, n_fft, win, return_complex=True))
    nf, T = X.shape[1], X.shape[2]
    X = X.reshape(B, S, nf, T, 2).permute(0, 2, 1, 3, 4).reshape(B, nf * S, T, 2)          # b (f s) t c
    x = X.permute(0, 2, 1, 3).reshape(B, T, nf * S * 2)                                     # b t (f s c)
    dims = [2 * f * S for f in bands]
    x = torch.stack([F.linear(_rms(xi, P[f"band_split.to_features.{i}.0.gamma"]), P[f"band_split.to_features.{i}.1.weight"],
                              P[f"band_split.to_features.{i}.1.bias"]) for i, xi in enumerate(x.split(dims, -1))], -2)
    nb = len(bands)
    rope = RotaryEmbedding(cfg.get("dim_head", 64))
    for i in range(cfg["depth"]):
        x = x.permute(0, 2, 1, 3).reshape(B * nb, T, dim)
        x = _transformer(P, f"layers.{i}.0", x, cfg.get("time_transformer_depth", 2), heads, rope)
        x = x.reshape(B, nb, T, dim).permute(0, 2, 1, 3).reshape(B * T, nb, dim)
        x = _transformer(P, f"layers.{i}.1", x, cfg.get("freq_transformer_depth", 2), heads, rope)
        x = x.reshape(B, T, nb, dim)
    x = _rms(x, P["final_norm.gamma"])
    depth = cfg.get("mask_estimator_depth", 2)
    outs = []
    for i in range(nb):
        h = x[..., i, :]
        for k in range(depth):
            p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
            h = F.linear(h, P[p + ".weight"], P[p + ".bias"])
            if k < depth - 1:
                h = torch.tanh(h)
        outs.append(F.glu(h, dim=-1))
    mask = torch.cat(outs, -1).reshape(B, T, nf * S, 2).permute(0, 2, 1, 3)                 # b (f s) t c
    Y = torch.view_as_complex(X.contiguous()) * torch.view_as_complex(mask.contiguous())
    Y = Y.reshape(B, nf, S, T).permute(0, 2, 1, 3).reshape(B * S, nf, T)
    out = torch.istft(Y, n_fft, hop, n_fft, win, return_complex=False)
    return out.reshape(B, S, -1)


def demix_windows(c=CHUNK):
    fade = c // 10
    fadein, fadeout = torch.linspace(0, 1, fade), torch.linspace(1, 0, fade)
    start, middle, finish = torch.ones(c), torch.ones(c), torch.ones(c)
    start[-fade:] *= fadeout
    finish[:fade] *= fadein
    middle[-fade:] *= fadeout
    middle[:fade] *= fadein
    return start, middle, finish


@torch.no_grad()
def demix_track(net_fn, mix, c=CHUNK, batch_size=4):
    """SeparateMDXC.demix_track with net_fn in place of the model: mix [S, L] fp32 -> {"vocals": np.ndarray [S, L]}.
    One chunk step (no overlap, no border pad); the last chunk is reflect-padded when longer than c // 2 + 1, else
    zero-padded; each batch's fade window is chosen from its last chunk and applied to every chunk of the batch."""
    w_start, w_middle, w_finish = demix_windows(c)
    n = mix.shape[1]
    result = torch.zeros((1,) + tuple(mix.shape))
    counter = torch.zeros((1,) + tuple(mix.shape))
    i, data, locs = 0, [], []
    while i < n:
        part = mix[:, i:i + c]
        length = part.shape[-1]
        if length < c:
            if length > c // 2 + 1:
                part = F.pad(part, (0, c - length), mode="reflect")
            else:
                part = F.pad(part, (0, c - length, 0, 0), mode="constant", value=0)
        data.append(part)
        locs.append((i, length))
        i += c
        if len(data) >= batch_size or i >= n:
            x = net_fn(torch.stack(data, 0))
            window = w_middle
            if i - c == 0:
                window = w_start
            elif i >= n:
                window = w_finish
            for j, (s, l) in enumerate(locs):
                result[..., s:s + l] += x[j][..., :l] * window[..., :l]
                counter[..., s:s + l] += window[..., :l]
            data, locs = [], []
    est = (result / counter).numpy()
    np.nan_to_num(est, copy=False, nan=0.0)
    return {"vocals": est[0]}
