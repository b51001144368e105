"""The UVR5 MDX23C oracle: the seeded parameters of TFC_TDF_net (lib_v5/vr_network/tfc_tdf_v3.py), the test audio,
SeparateMDXC.demix_track (uvr5/separate.py:492-574) restated with the chunk length and the target axis as parameters, and
TFC_TDF_net.forward restated in stock torch for the benchmark's stock-PyTorch arms.  The goldens come from the unmodified
reference module (oracle/pin_mdx23c.py imports it and checks this file against it)."""
import copy
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

from oracle.bs_roformer_oracle import demix_windows, make_audio  # noqa: F401  (make_audio: the shared test audio)

# The published 8K-FFT InstVoc HQ configuration, written from memory (no checkpoint or YAML was at hand to confirm it).
DEFAULT = {
    "audio": {"chunk_size": 261120, "dim_f": 4096, "dim_t": 256, "hop_length": 1024, "n_fft": 8192, "num_channels": 2,
              "sample_rate": 44100, "min_mean_abs": 0.001},
    "model": {"act": "gelu", "bottleneck_factor": 4, "growth": 128, "norm": "InstanceNorm", "num_blocks_per_scale": 2,
              "num_channels": 128, "num_scales": 5, "num_subbands": 4, "scale": [2, 2]},
    "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": None},
}


def config(over):
    """DEFAULT with the nested overrides `over` ({"audio": {...}, ...})"""
    cfg = copy.deepcopy(DEFAULT)
    for sec, fields in over.items():
        cfg[sec].update(fields)
    return cfg


def namespace(cfg):
    """nested dict -> nested SimpleNamespace (the attribute access TFC_TDF_net uses)"""
    return SimpleNamespace(**{k: namespace(v) if isinstance(v, dict) else v for k, v in cfg.items()})


def param_spec(cfg):
    """-> {state_dict key: shape} of TFC_TDF_net(cfg), in the reference's key order."""
    m, a = cfg["model"], cfg["audio"]
    k, n, l, c, g, bn = (m["num_subbands"], m["num_scales"], m["num_blocks_per_scale"], m["num_channels"], m["growth"],
                         m["bottleneck_factor"])
    nt = 1 if cfg["training"]["target_instrument"] else len(cfg["training"]["instruments"])
    D, f = 2 * k * a["num_channels"], a["dim_f"] // k

    def tfc_tdf(p, in_c, c, f):
        out = {}
        for j in range(l):
            q = f"{p}.blocks.{j}"
            out.update({q + ".tfc1.0.weight": (in_c,), q + ".tfc1.0.bias": (in_c,), q + ".tfc1.2.weight": (c, in_c, 3, 3),
                        q + ".tdf.0.weight": (c,), q + ".tdf.0.bias": (c,), q + ".tdf.2.weight": (f // bn, f),
                        q + ".tdf.3.weight": (c,), q + ".tdf.3.bias": (c,), q + ".tdf.5.weight": (f, f // bn),
                        q + ".tfc2.0.weight": (c,), q + ".tfc2.0.bias": (c,), q + ".tfc2.2.weight": (c, c, 3, 3),
                        q + ".shortcut.weight": (c, in_c, 1, 1)})
            in_c = c
        return out

    spec = {"first_conv.weight": (c, D, 1, 1)}
    for i in range(n):
        spec.update(tfc_tdf(f"encoder_blocks.{i}.tfc_tdf", c, c, f))
        p = f"encoder_blocks.{i}.downscale.conv"
        spec.update({p + ".0.weight": (c,), p + ".0.bias": (c,), p + ".2.weight": (c + g, c, 2, 2)})
        f, c = f // 2, c + g
    spec.update(tfc_tdf("bottleneck_block", c, c, f))
    for i in range(n):
        p = f"decoder_blocks.{i}.upscale.conv"
        spec.update({p + ".0.weight": (c,), p + ".0.bias": (c,), p + ".2.weight": (c, c - g, 2, 2)})
        f, c = f * 2, c - g
        spec.update(tfc_tdf(f"decoder_blocks.{i}.tfc_tdf", 2 * c, c, f))
    spec.update({"final_conv.0.weight": (c, c + D, 1, 1), "final_conv.2.weight": (nt * D, c, 1, 1)})
    return spec


def init_params(spec, seed):
    """Seeded weights: conv and Linear weights N(0, 1 / fan_in) (a transposed conv's fan-in is its input channels), norm
    weights in [0.5, 1.5], norm biases N(0, 0.1^2)."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for key, shape in spec.items():
        if len(shape) == 1:
            P[key] = (0.5 + torch.rand(shape, generator=g)) if key.endswith("weight") else 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = shape[0] if ".upscale." in key else int(np.prod(shape[1:]))
            P[key] = torch.randn(shape, generator=g) / fan_in ** 0.5
    return P


@torch.no_grad()
def demix_track(net_fn, mix, c, batch_size=4):
    """SeparateMDXC.demix_track with net_fn in place of the model and chunk length c: mix [S, L] fp32 ->
    {"vocals": est[0], "other": est[1]} over the estimate [n_targets, S, L] (one target: {"vocals": [S, L]}).  The
    reference's loop with its buffers given the target axis: one chunk step (no overlap, no border pad); the last chunk is
    reflect-padded when longer than c // 2 + 1, else zero-padded; each batch's fade window is chosen from its last chunk."""
    w_start, w_middle, w_finish = demix_windows(c)
    S, n = mix.shape
    result = counter = None
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
            x = x.reshape(x.shape[0], -1, S, x.shape[-1])             # [chunks, targets, S, c]
            if result is None:
                result = torch.zeros((x.shape[1], S, n))
                counter = torch.zeros((x.shape[1], S, n))
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
    return {k: v for k, v in zip(["vocals", "other"], est)}


def _norm_act(P, p, x):
    return F.gelu(F.instance_norm(x, weight=P[p + ".weight"], bias=P[p + ".bias"], eps=1e-5))


def _tfc_tdf(P, p, x, l):
    for j in range(l):
        q = f"{p}.blocks.{j}"
        s = F.conv2d(x, P[q + ".shortcut.weight"])
        x = F.conv2d(_norm_act(P, q + ".tfc1.0", x), P[q + ".tfc1.2.weight"], padding=1)
        t = F.linear(_norm_act(P, q + ".tdf.0", x), P[q + ".tdf.2.weight"])
        x = x + F.linear(_norm_act(P, q + ".tdf.3", t), P[q + ".tdf.5.weight"])
        x = F.conv2d(_norm_act(P, q + ".tfc2.0", x), P[q + ".tfc2.2.weight"], padding=1)
        x = x + s
    return x


def forward(P, cfg, raw):
    """TFC_TDF_net(cfg).forward(raw) in stock torch (the stock-PyTorch arm of tools/bench_uvr5.py --net mdx23c): raw
    [B, S, L] -> [B, n_targets, S, hop * (L // hop)], or [B, S, ...] for one target (the [B, S, ...] a mono model means;
    the reference's own last reshape assumes two channels)"""
    a, m = cfg["audio"], cfg["model"]
    n_fft, hop, dim_f, k = a["n_fft"], a["hop_length"], a["dim_f"], m["num_subbands"]
    n, l = m["num_scales"], m["num_blocks_per_scale"]
    nt = 1 if cfg["training"]["target_instrument"] else len(cfg["training"]["instruments"])
    B, S, L = raw.shape
    NB = n_fft // 2 + 1
    win = torch.hann_window(n_fft, device=raw.device)
    X = torch.view_as_real(torch.stft(raw.reshape(-1, L), n_fft, hop, window=win, center=True, return_complex=True))
    X = X.permute(0, 3, 1, 2).reshape(B, S * 2, NB, -1)[..., :dim_f, :]
    mix = x = X.reshape(B, S * 2 * k, dim_f // k, -1)
    first = x = F.conv2d(x, P["first_conv.weight"])
    x = x.transpose(-1, -2)
    enc = []
    for i in range(n):
        x = _tfc_tdf(P, f"encoder_blocks.{i}.tfc_tdf", x, l)
        enc.append(x)
        p = f"encoder_blocks.{i}.downscale.conv"
        x = F.conv2d(_norm_act(P, p + ".0", x), P[p + ".2.weight"], stride=2)
    x = _tfc_tdf(P, "bottleneck_block", x, l)
    for i in range(n):
        p = f"decoder_blocks.{i}.upscale.conv"
        x = F.conv_transpose2d(_norm_act(P, p + ".0", x), P[p + ".2.weight"], stride=2)
        x = _tfc_tdf(P, f"decoder_blocks.{i}.tfc_tdf", torch.cat([x, enc.pop()], 1), l)
    x = x.transpose(-1, -2) * first
    x = F.conv2d(F.gelu(F.conv2d(torch.cat([mix, x], 1), P["final_conv.0.weight"])), P["final_conv.2.weight"])
    t = x.shape[-1]
    x = x.reshape(B, nt, S * 2, k, dim_f // k, t).reshape(B, nt, S * 2, dim_f, t)
    x = torch.cat([x, x.new_zeros(B, nt, S * 2, NB - dim_f, t)], 3).reshape(B * nt * S, 2, NB, t)
    out = torch.istft(torch.complex(x[:, 0].float(), x[:, 1].float()), n_fft, hop, window=win, center=True)
    return out.reshape(B, nt, S, -1) if nt > 1 else out.reshape(B, S, -1)
