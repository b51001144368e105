"""CPU restatement of the UVR5 Mel-Band Roformer: MelBandRoformer.forward in eval mode (lib_v5/vr_network/mel_band_roformer.py:
244-478, attend.py), in stock torch fp32 with seeded weights, driven chunk by chunk by SeparateMDXC.demix_track (the
BS-Roformer oracle's restatement of it).

Key names are the reference's state_dict names.  Dropout is the identity.  The band tables follow the reference's own steps
(filterbank > 0, repeat / boolean-mask indexing, stereo interleave 2f + s) on top of oracle/mel_oracle.py's restatement of
librosa.filters.mel.  The rotary embedding is oracle/bs_roformer_oracle.py's stand-in.  `import_reference` loads the
unmodified reference module for oracle/pin_mel_roformer.py, which checks this file against it."""
import importlib
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle import bs_roformer_oracle as BR
from oracle import mel_oracle

# the widely distributed vocal model's configuration (44.1 kHz, 60 bands, dim 384, depth 6)
DEFAULT = dict(
    attn_dropout=0.1, depth=6, dim=384, dim_freqs_in=1025, dim_head=64, ff_dropout=0.1, flash_attn=True,
    freq_transformer_depth=1, heads=8, mask_estimator_depth=2, match_input_audio_length=False, multi_stft_hop_size=147,
    multi_stft_normalized=False, multi_stft_resolution_loss_weight=1.0,
    multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256), num_bands=60, num_stems=1, sample_rate=44100,
    stereo=True, stft_hop_length=441, stft_n_fft=2048, stft_normalized=False, stft_win_length=2048, time_transformer_depth=1,
)
CHUNK = BR.CHUNK
init_params, make_audio, demix_track = BR.init_params, BR.make_audio, BR.demix_track


def band_tables(sr, n_fft, num_bands, stereo):
    """mel_band_roformer.py:314-340 -> (freq_indices, num_freqs_per_band, num_bands_per_freq) as int64 tensors; freq_indices
    indexes the '(f s)' axis (2 f + s when stereo)"""
    fb = torch.from_numpy(mel_oracle.mel_filterbank(sr, n_fft, num_bands))
    fb[0][0] = 1.0
    fb[-1, -1] = 1.0
    member = fb > 0
    assert member.any(dim=0).all(), "all frequencies need to be covered by all bands for now"
    freq_indices = torch.arange(n_fft // 2 + 1)[None, :].expand(num_bands, -1)[member]
    if stereo:
        freq_indices = (freq_indices[:, None] * 2 + torch.arange(2)).reshape(-1)
    return freq_indices, member.sum(1), member.sum(0)


def param_spec(cfg):
    """-> {state_dict key: shape} of MelBandRoformer(**cfg) (one stem), in the reference's key order"""
    dim, heads, dh = cfg["dim"], cfg.get("heads", 8), cfg.get("dim_head", 64)
    inner, S = heads * dh, 2 if cfg.get("stereo", False) else 1
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
            spec[f"layers.{i}.{a}.norm.gamma"] = (dim,)
    _, per_band, _ = band_tables(cfg.get("sample_rate", 44100), cfg.get("stft_n_fft", 2048), cfg.get("num_bands", 60), S == 2)
    dims = [2 * int(n) * S for n in per_band]
    for i, d in enumerate(dims):
        spec[f"band_split.to_features.{i}.0.gamma"] = (d,)
        spec[f"band_split.to_features.{i}.1.weight"] = (dim, d)
        spec[f"band_split.to_features.{i}.1.bias"] = (dim,)
    depth, hid = cfg.get("mask_estimator_depth", 1) + 1, 4 * dim         # MLP(depth) holds depth + 1 Linears here
    for i, d in enumerate(dims):
        io = [dim] + [hid] * (depth - 1) + [2 * d]
        for k in range(depth):
            p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
            spec[p + ".weight"] = (io[k + 1], io[k])
            spec[p + ".bias"] = (io[k + 1],)
    return spec


@torch.no_grad()
def forward(P, cfg, raw):
    """MelBandRoformer(**cfg).forward(raw) in eval mode: raw [B, S, L] (or [B, L] mono) fp32 -> [B, S, hop * (L // hop)]
    ([B, S, L] with match_input_audio_length)"""
    if raw.dim() == 2:
        raw = raw[:, None]
    B, S, L = raw.shape
    n_fft, hop, dim = cfg["stft_n_fft"], cfg["stft_hop_length"], cfg["dim"]
    heads, nb = cfg.get("heads", 8), cfg.get("num_bands", 60)
    fi, per_band, per_bin = band_tables(cfg.get("sample_rate", 44100), n_fft, nb, S == 2)
    win = torch.hann_window(n_fft, device=raw.device)
    X = torch.view_as_real(torch.stft(raw.reshape(B * S, L), n_fft, hop, n_fft, win, return_complex=True))
    nf, T = X.shape[1], X.shape[2]
    X = X.reshape(B, S, nf, T, 2).permute(0, 2, 1, 3, 4).reshape(B, nf * S, T, 2)          # b (f s) t c
    x = X[:, fi.to(raw.device)].permute(0, 2, 1, 3).reshape(B, T, -1)                       # b t (f c)
    dims = [2 * int(n) * S for n in per_band]
    x = torch.stack([F.linear(BR._rms(xi, P[f"band_split.to_features.{i}.0.gamma"]), P[f"band_split.to_features.{i}.1.weight"],
                              P[f"band_split.to_features.{i}.1.bias"]) for i, xi in enumerate(x.split(dims, -1))], -2)
    rope = BR.RotaryEmbedding(cfg.get("dim_head", 64))
    for i in range(cfg["depth"]):
        x = x.permute(0, 2, 1, 3).reshape(B * nb, T, dim)
        x = BR._transformer(P, f"layers.{i}.0", x, cfg.get("time_transformer_depth", 2), heads, rope)
        x = BR._rms(x, P[f"layers.{i}.0.norm.gamma"])
        x = x.reshape(B, nb, T, dim).permute(0, 2, 1, 3).reshape(B * T, nb, dim)
        x = BR._transformer(P, f"layers.{i}.1", x, cfg.get("freq_transformer_depth", 2), heads, rope)
        x = BR._rms(x, P[f"layers.{i}.1.norm.gamma"])
        x = x.reshape(B, T, nb, dim)
    depth = cfg.get("mask_estimator_depth", 1) + 1
    outs = []
    for i in range(nb):
        h = x[..., i, :]
        for k in range(depth):
            p = f"mask_estimators.0.to_freqs.{i}.0.{2 * k}"
            h = F.linear(h, P[p + ".weight"], P[p + ".bias"])
            if k < depth - 1:
                h = torch.tanh(h)
        outs.append(F.glu(h, dim=-1))
    m = torch.view_as_complex(torch.cat(outs, -1).reshape(B, T, -1, 2).permute(0, 2, 1, 3).contiguous())   # b f' t
    summed = torch.zeros(B, nf * S, T, dtype=m.dtype, device=m.device).index_add_(1, fi.to(m.device), m)
    avg = summed / per_bin.repeat_interleave(S).to(m.device)[:, None].clamp(min=1e-8)
    Y = torch.view_as_complex(X.contiguous()) * avg
    Y = Y.reshape(B, nf, S, T).permute(0, 2, 1, 3).reshape(B * S, nf, T)
    out = torch.istft(Y, n_fft, hop, n_fft, win, return_complex=False,
                      length=L if cfg.get("match_input_audio_length", False) else None)
    return out.reshape(B, S, -1)


def import_reference():
    """-> (the reference's unmodified mel_band_roformer module, uvr5 separate module).  Shims: `attend` (imported without its
    package) is the reference's own attend module; rotary_embedding_torch.RotaryEmbedding is bs_roformer_oracle's stand-in;
    librosa.filters.mel is mel_oracle's restatement.  Needs EVK_REFERENCE."""
    from oracle.pin_uvr5 import import_reference as import_uvr5
    from oracle.ref_import import _stub
    _, separate = import_uvr5()
    sys.modules["attend"] = importlib.import_module("src.audiokit.uvr5.lib_v5.vr_network.attend")
    filt = _stub("librosa.filters", mel=lambda sr, n_fft, n_mels=128, fmin=0.0, fmax=None, **_:
                 mel_oracle.mel_filterbank(sr, n_fft, n_mels, fmin, fmax))
    sys.modules["librosa"].filters = filt
    sys.modules["rotary_embedding_torch"].RotaryEmbedding = BR.RotaryEmbedding
    mod = importlib.import_module("src.audiokit.uvr5.lib_v5.vr_network.mel_band_roformer")
    mod.RotaryEmbedding = BR.RotaryEmbedding
    return mod, separate
