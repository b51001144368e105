"""Float64 emulation of BS-Roformer and Mel-Band Roformer under a float16 / bfloat16 compute type, as bs_roformer.py runs
them: both operands of every Linear (qkv and gates, to_out, the feed-forward pair, band split, mask MLPs) rounded to nearest
even to 16 bits, and in the attention the rotated q and k, v and the softmax probabilities P rounded the same way.  The
activation is rounded from its fp32 value; the weight after the RMSNorm gamma * sqrt(dim) before it is folded into its
columns, as the library packs it.  Softmax sums, the gate, the norms, the GLU, the STFT and the iSTFT are float64.  With
dtype None nothing is rounded, and the computation is the float64 restatement of oracle/bs_roformer_oracle.py and
oracle/mel_roformer_oracle.py."""
import math

import torch
import torch.nn.functional as F

from oracle import bs_roformer_oracle as BR
from oracle import mel_roformer_oracle as MR


def rounding(dtype):
    """-> h: x rounded to fp32, then to nearest even in `dtype`, as float64; the identity when dtype is None"""
    if dtype is None:
        return lambda x: x
    return lambda x: x.float().to(dtype).double()


def lin(h, x, w, b=None, gamma=None):
    """h(x) h(W)^T + b; with gamma, the RMSNorm before the Linear folded as the library does: h(x / ||x||) h(W gamma sqrt(d))^T"""
    if gamma is not None:
        x = F.normalize(x, dim=-1)
        w = w * (gamma * math.sqrt(gamma.numel()))[None, :]
    y = h(x) @ h(w).T
    return y if b is None else y + b


def rotate(x, cs):
    """interleaved rotary embedding of x [..., L, 64] by cs [L, 32, 2] (cos, sin)"""
    c, s = cs[..., 0].repeat_interleave(2, -1), cs[..., 1].repeat_interleave(2, -1)
    y = x.unflatten(-1, (-1, 2))
    return x * c + torch.stack((-y[..., 1], y[..., 0]), -1).flatten(-2) * s


def attention(h, qkv, gates, heads, cs, block=64):
    """qkv [n, L, 3 heads 64], gates [n, L, heads] -> [n, L, heads 64]: h(rot q) h(rot k)^T / 8, p = exp(s - max),
    o = h(p) h(v) / sum(p) * sigmoid(gate); sequences in blocks of `block` to bound the [L, L] scores' memory"""
    n, L, _ = qkv.shape
    out = torch.empty((n, L, heads * 64), dtype=qkv.dtype, device=qkv.device)
    for u in range(0, n, block):
        qq, kk, vv = qkv[u:u + block].reshape(-1, L, 3, heads, 64).permute(2, 0, 3, 1, 4)
        q, k, v = h(rotate(qq, cs[:L])), h(rotate(kk, cs[:L])), h(vv)
        s = q @ k.transpose(-1, -2) / 8.0
        p = torch.exp(s - s.amax(-1, keepdim=True))
        o = (h(p) @ v) / p.sum(-1, keepdim=True) * torch.sigmoid(gates[u:u + block]).permute(0, 2, 1)[..., None]
        out[u:u + block] = o.permute(0, 2, 1, 3).reshape(-1, L, heads * 64)
    return out


def transformer(h, P, p, x, depth, heads, cs):
    """the `depth` Attention + FeedForward layers at prefix p on x [n, L, dim]"""
    for j in range(depth):
        q = f"{p}.layers.{j}"
        g = P[q + ".0.norm.gamma"]
        qkv = lin(h, x, P[q + ".0.to_qkv.weight"], gamma=g)
        gates = lin(h, x, P[q + ".0.to_gates.weight"], P[q + ".0.to_gates.bias"], gamma=g)
        x = lin(h, attention(h, qkv, gates, heads, cs), P[q + ".0.to_out.0.weight"]) + x
        f = F.gelu(lin(h, x, P[q + ".1.net.1.weight"], P[q + ".1.net.1.bias"], gamma=P[q + ".1.net.0.gamma"]))
        x = lin(h, f, P[q + ".1.net.4.weight"], P[q + ".1.net.4.bias"]) + x
    return x


def cos_sin(L, device):
    """the fp32 rotary table both the oracle and the library use, [L, 32, 2] in float64"""
    c, s = BR.rotary_cos_sin(L)
    return torch.stack([c, s], -1).double().to(device)


@torch.no_grad()
def forward(P, cfg, raw, dtype, mel=False):
    """BSRoformer(**cfg) (mel False) or MelBandRoformer(**cfg) forward of raw [B, S, L] (or [B, L] mono) with the 16-bit
    contract of `dtype` (None: unrounded), in float64 on raw's device -> [B, S, hop * (L // hop)] ([B, S, L] for a Mel-Band
    model with match_input_audio_length)"""
    h = rounding(dtype)
    dev = raw.device
    P = {k: v.double().to(dev) for k, v in P.items()}
    if raw.dim() == 2:
        raw = raw[:, None]
    raw = raw.double()
    B, S, L = raw.shape
    n_fft, hop, dim, heads = cfg["stft_n_fft"], cfg["stft_hop_length"], cfg["dim"], cfg.get("heads", 8)
    win = torch.hann_window(n_fft, dtype=torch.float64, device=dev)
    X = torch.view_as_real(torch.stft(raw.reshape(B * S, L), n_fft, hop, n_fft, win, return_complex=True))
    nf, T = X.shape[1], X.shape[2]
    X = X.reshape(B, S, nf, T, 2).permute(0, 2, 1, 3, 4).reshape(B, nf * S, T, 2)          # b (f s) t c
    if mel:
        nb = cfg.get("num_bands", 60)
        fi, per_band, per_bin = MR.band_tables(cfg.get("sample_rate", 44100), n_fft, nb, S == 2)
        x = X[:, fi.to(dev)].permute(0, 2, 1, 3).reshape(B, T, -1)
        dims = [2 * int(n) * S for n in per_band]
        n_lin, last_norm = cfg.get("mask_estimator_depth", 1) + 1, f"layers.{cfg['depth'] - 1}.1.norm.gamma"
    else:
        nb = len(cfg["freqs_per_bands"])
        x = X.permute(0, 2, 1, 3).reshape(B, T, nf * S * 2)
        dims = [2 * f * S for f in cfg["freqs_per_bands"]]
        n_lin, last_norm = cfg.get("mask_estimator_depth", 2), "final_norm.gamma"
    x = torch.stack([lin(h, xi, P[f"band_split.to_features.{i}.1.weight"], P[f"band_split.to_features.{i}.1.bias"],
                         gamma=P[f"band_split.to_features.{i}.0.gamma"]) for i, xi in enumerate(x.split(dims, -1))], -2)
    cs_t, cs_f = cos_sin(T, dev), cos_sin(nb, dev)
    for i in range(cfg["depth"]):
        x = x.permute(0, 2, 1, 3).reshape(B * nb, T, dim)
        x = transformer(h, P, f"layers.{i}.0", x, cfg.get("time_transformer_depth", 2), heads, cs_t)
        if mel:
            x = BR._rms(x, P[f"layers.{i}.0.norm.gamma"])
        x = x.reshape(B, nb, T, dim).permute(0, 2, 1, 3).reshape(B * T, nb, dim)
        x = transformer(h, P, f"layers.{i}.1", x, cfg.get("freq_transformer_depth", 2), heads, cs_f)
        if mel and i < cfg["depth"] - 1:
            x = BR._rms(x, P[f"layers.{i}.1.norm.gamma"])
        x = x.reshape(B, T, nb, dim)
    outs = []
    for i in range(nb):                                    # the last norm's gamma is folded into each mask MLP's first Linear
        hc = x[..., i, :]
        for k in range(n_lin):
            p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
            hc = lin(h, hc, P[p + ".weight"], P[p + ".bias"], gamma=P[last_norm] if k == 0 else None)
            if k < n_lin - 1:
                hc = torch.tanh(hc)
        outs.append(F.glu(hc, dim=-1))
    m = torch.view_as_complex(torch.cat(outs, -1).reshape(B, T, -1, 2).permute(0, 2, 1, 3).contiguous())
    if mel:
        summed = torch.zeros(B, nf * S, T, dtype=m.dtype, device=dev).index_add_(1, fi.to(dev), m)
        m = summed / per_bin.repeat_interleave(S).to(dev)[:, None].double().clamp(min=1e-8)
    Y = torch.view_as_complex(X.contiguous()) * m
    Y = Y.reshape(B, nf, S, T).permute(0, 2, 1, 3).reshape(B * S, nf, T)
    length = L if mel and cfg.get("match_input_audio_length", False) else None
    return torch.istft(Y, n_fft, hop, n_fft, win, return_complex=False, length=length).reshape(B, S, -1)


def demix_track(P, cfg, mix, dtype, mel=False, device="cpu"):
    """SeparateMDXC.demix_track (oracle/bs_roformer_oracle.py) with the emulated forward on `device` -> {"vocals": [S, n]}"""
    net = lambda chunks: forward(P, cfg, chunks.to(device), dtype, mel).cpu()           # noqa: E731
    return BR.demix_track(net, mix)
