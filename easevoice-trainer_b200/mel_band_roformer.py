"""UVR5 Mel-Band Roformer vocal separation on the library's kernels: the MelBandRoformer of
lib_v5/vr_network/mel_band_roformer.py:244-478 (inference), run chunk by chunk through bs_roformer.demix_track.

It is the BS-Roformer (bs_roformer.AxialRoformer: the same rotary gated axial attention, GELU feed-forward, band and mask
Linears and folded weights) with three differences:
  * the bands are the non-zero bins of the rows of a Slaney mel filterbank (mel_processing.slaney_filterbank, the
    restatement of librosa.filters.mel, with its first and last weight forced to 1), so adjacent bands share bins.
    evk_band_input gathers each band's bins through a device bin table and L2-normalises its segment;
  * each band's mask covers its own bins.  evk_melband_mask_avg sums the bands covering a bin in ascending band order and
    divides by their count (the reference's scatter_add_ / num_bands_per_freq), into the mask layout the inverse STFT takes;
  * every Transformer ends in its own RMSNorm and there is no final norm.  Those norms sit on the residual stream between
    transformers, so they run as evk_row_norm with their gamma, except the last, which feeds only the mask estimators and
    is folded into their first Linear like every other RMSNorm.
"""
import re

import numpy as np
import torch

from .bs_roformer import AxialRoformer, check_sizes, check_stft
from .mel_processing import slaney_filterbank

# The widely distributed Mel-Band Roformer vocal model's configuration (44.1 kHz, 60 bands, dim 384, depth 6).
DEFAULT_CONFIG = dict(
    attn_dropout=0.1, depth=6, dim=384, dim_freqs_in=1025, dim_head=64, ff_dropout=0.1, flash_attn=True,
    freq_transformer_depth=1, heads=8, mask_estimator_depth=2, match_input_audio_length=False, multi_stft_hop_size=147,
    multi_stft_normalized=False, multi_stft_resolution_loss_weight=1.0,
    multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256), num_bands=60, num_stems=1, sample_rate=44100,
    stereo=True, stft_hop_length=441, stft_n_fft=2048, stft_normalized=False, stft_win_length=2048, time_transformer_depth=1,
)


def band_tables(sample_rate, n_fft, num_bands):
    """The reference's band layout (mel_band_roformer.py:312-340) -> (bins, band_off, cover, cover_off): band i holds the
    bins bins[band_off[i]:band_off[i+1]] (ascending), and bin f is held by the slots cover[cover_off[f]:cover_off[f+1]] of
    `bins` (ascending, that is in band order).  ValueError when a bin is in no band or a band has no bin."""
    fb = slaney_filterbank(sample_rate, n_fft, num_bands)
    fb[0, 0] = 1.0
    fb[-1, -1] = 1.0
    member = fb > 0
    if not member.any(0).all():
        raise ValueError(f"the mel filterbank (sample_rate {sample_rate}, n_fft {n_fft}, num_bands {num_bands}) leaves bins "
                         f"{np.nonzero(~member.any(0))[0][:5].tolist()} in no band: all frequencies need to be covered")
    per_band = member.sum(1)
    if (per_band == 0).any():
        raise ValueError(f"the mel filterbank (sample_rate {sample_rate}, n_fft {n_fft}, num_bands {num_bands}) has bands "
                         f"{np.nonzero(per_band == 0)[0][:5].tolist()} with no bins")
    bins = np.nonzero(member)[1].astype(np.int32)                                     # row-major: band by band
    band_off = np.concatenate([[0], np.cumsum(per_band)]).astype(np.int32)
    cover = np.argsort(bins, kind="stable").astype(np.int32)
    cover_off = np.concatenate([[0], np.cumsum(member.sum(0))]).astype(np.int32)
    return bins, band_off, cover, cover_off


class MelBandRoformer(AxialRoformer):
    """MelBandRoformer(**config) for inference on CUDA.  Takes the reference's keyword arguments; the training-only ones
    (`*_dropout`, `multi_stft_*`, `flash_attn`) and dim_freqs_in (the reference ignores it too) are accepted and ignored.
    Raises ValueError for what the kernels do not take: dim_head != 64, num_stems != 1, stft_n_fft not a power of two in
    [256, 4096], stft_win_length != stft_n_fft, stft_normalized, a custom stft_window_fn, a hop above n_fft / 2, and a mel
    filterbank that leaves a bin in no band or a band with no bins."""

    def __init__(self, dim, *, depth, stereo=False, num_stems=1, time_transformer_depth=2, freq_transformer_depth=2,
                 num_bands=60, dim_head=64, heads=8, attn_dropout=0.1, ff_dropout=0.1, flash_attn=True, dim_freqs_in=1025,
                 sample_rate=44100, stft_n_fft=2048, stft_hop_length=512, stft_win_length=2048, stft_normalized=False,
                 stft_window_fn=None, mask_estimator_depth=1, multi_stft_resolution_loss_weight=1.0,
                 multi_stft_resolutions_window_sizes=(4096, 2048, 1024, 512, 256), multi_stft_hop_size=147,
                 multi_stft_normalized=False, multi_stft_window_fn=None, match_input_audio_length=False):
        if dim_head != 64:
            raise ValueError(f"dim_head must be 64, got {dim_head}")
        if num_stems != 1:
            raise ValueError(f"num_stems must be 1, got {num_stems}")
        n_fft = check_stft(stft_n_fft, stft_win_length, stft_hop_length, stft_normalized, stft_window_fn)
        if num_bands < 1:
            raise ValueError(f"num_bands must be >= 1, got {num_bands}")
        tables = band_tables(sample_rate, n_fft, int(num_bands))
        if mask_estimator_depth < 0:
            raise ValueError(f"mask_estimator_depth must be >= 0, got {mask_estimator_depth}")
        check_sizes(dim, heads, depth, mask_estimator_depth + 1)
        # the reference's MLP here has mask_estimator_depth hidden layers: one Linear more than BS-Roformer's
        super().__init__(dim, depth, heads, stereo, time_transformer_depth, freq_transformer_depth, n_fft, stft_hop_length,
                         mask_estimator_depth, mask_estimator_depth + 1, *tables,
                         match_input_audio_length=match_input_audio_length)
        self.num_bands, self.sample_rate = int(num_bands), int(sample_rate)

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _dims_in(self):
        return [2 * self.S * int(n) for n in np.diff(self.band_off)]

    def state_dict_shapes(self):
        """-> {key: shape} of the reference's MelBandRoformer(**config).state_dict() (rotary modules hold no state there)"""
        spec = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                spec.update(self._layer_shapes(f"layers.{i}.{a}", n))
                spec[f"layers.{i}.{a}.norm.gamma"] = (self.dim,)
        spec.update(self._band_shapes(self._dims_in()))
        return spec

    def _last_norm(self):
        return f"layers.{self.depth - 1}.1.norm.gamma"

    def _fold(self, sd):
        """As BSRoformer's, with each Transformer's output-norm gamma kept as a device vector (`<prefix>.norm.g`) except the
        last one's, which is folded into the first Linear of every mask MLP"""
        out = {}
        for i in range(self.depth):
            for a, n in ((0, self.t_depth), (1, self.f_depth)):
                p = f"layers.{i}.{a}"
                self._fold_layers(sd, p, n, out)
                if p + ".norm.gamma" != self._last_norm():
                    out[p + ".norm.g"] = sd[p + ".norm.gamma"].contiguous()
        self._fold_bands(sd, self.num_bands, sd[self._last_norm()], out)
        return out

    @classmethod
    def infer_config(cls, sd, **config):
        """The constructor arguments that a reference state_dict determines: dim and num_bands from band_split, heads from
        to_gates, dim_head from to_qkv, depth and the time / frequency depths from the layer keys, mask_estimator_depth from the
        mask MLP keys, and stereo and stft_n_fft by matching the band input widths against the filterbank of every power of
        two n_fft in [256, 4096] at the sample rate (each fixed by the caller when given).  Everything else comes from
        DEFAULT_CONFIG unless the caller gives it.  ValueError when the weights match no configuration, or more than one."""
        cfg = dict(DEFAULT_CONFIG)
        cfg.update(config)

        def count(pattern, step=1):
            idx = {int(m.group(1)) for k in sd for m in [re.fullmatch(pattern, k)] if m}
            if idx != set(range(0, step * len(idx), step)):
                raise ValueError(f"state_dict keys matching {pattern} are not numbered 0, {step}, ...: {sorted(idx)[:8]}")
            return len(idx)

        widths = []
        for i in range(count(r"band_split\.to_features\.(\d+)\.1\.weight")):
            w = sd.get(f"band_split.to_features.{i}.1.weight")
            g = sd.get(f"band_split.to_features.{i}.0.gamma")
            if w is None or g is None or w.dim() != 2 or g.dim() != 1:
                raise ValueError(f"band_split.to_features.{i}: missing or malformed weights")
            widths.append(int(g.shape[0]))
            dim = int(w.shape[0])
        if not widths:
            raise ValueError("state_dict has no band_split weights: not a MelBandRoformer checkpoint")
        gates = sd.get("layers.0.0.layers.0.0.to_gates.weight", sd.get("layers.0.1.layers.0.0.to_gates.weight"))
        qkv = sd.get("layers.0.0.layers.0.0.to_qkv.weight", sd.get("layers.0.1.layers.0.0.to_qkv.weight"))
        inferred = dict(dim=dim, num_bands=len(widths), depth=count(r"layers\.(\d+)\.0\.norm\.gamma"),
                        time_transformer_depth=count(r"layers\.0\.0\.layers\.(\d+)\.0\.to_qkv\.weight"),
                        freq_transformer_depth=count(r"layers\.0\.1\.layers\.(\d+)\.0\.to_qkv\.weight"),
                        mask_estimator_depth=count(r"mask_estimators\.0\.to_freqs\.0\.0\.(\d+)\.weight", 2) - 1)
        if gates is not None and qkv is not None:
            inferred["heads"] = int(gates.shape[0])
            inferred["dim_head"] = int(qkv.shape[0]) // (3 * inferred["heads"])
        cfg.update({k: v for k, v in inferred.items() if k not in config})
        n_ffts = [config["stft_n_fft"]] if "stft_n_fft" in config else [2 ** e for e in range(8, 13)]
        stereos = [bool(config["stereo"])] if "stereo" in config else [True, False]
        found = []
        for n_fft in n_ffts:
            try:
                _, off, _, _ = band_tables(cfg["sample_rate"], n_fft, len(widths))
            except ValueError:
                continue
            for st in stereos:
                if [2 * (2 if st else 1) * int(n) for n in np.diff(off)] == widths:
                    found.append((n_fft, st))
        if len(found) != 1:
            raise ValueError(f"the band_split widths match {'no' if not found else 'more than one'} (stft_n_fft, stereo) at "
                             f"sample_rate {cfg['sample_rate']} and {len(widths)} bands{': ' + str(found) if found else ''}; "
                             "pass stft_n_fft / stereo / sample_rate explicitly")
        n_fft, stereo = found[0]
        cfg.update(stft_n_fft=n_fft, stereo=stereo)
        if "stft_win_length" not in config:
            cfg["stft_win_length"] = n_fft
        cfg["dim_freqs_in"] = n_fft // 2 + 1
        return cfg

    @classmethod
    def from_pretrained(cls, path, device="cuda", compute_type=None, **config):
        """A MelBandRoformer with the weights of a reference checkpoint file, on `device`.  The configuration is inferred
        from the weight shapes (infer_config); sample_rate and stft_hop_length, which the weights do not determine, default
        to DEFAULT_CONFIG's (44.1 kHz, hop 441) and are the caller's to set, as is anything passed in `config`.
        compute_type: as set_compute_type."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        return cls(**cls.infer_config(sd, **config)).to(device).load_state_dict(sd).set_compute_type(compute_type)
