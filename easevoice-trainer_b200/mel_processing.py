"""Drop-in for /root/reference/src/easevoice/module/mel_processing.py (same function names, argument order and
[B, F, T] results), computed by the fused sm_90a mel kernel instead of torch.stft + matmul + elementwise ops.

The Slaney filterbank is librosa.filters.mel (librosa 0.9.2, the reference's pinned dependency) restated here in
float64 -> float32; librosa itself is not needed.
"""
import math

import numpy as np
import torch

from . import ops

MAX_WAV_VALUE = 32768.0
_banks = {}


def slaney_filterbank(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) (htk=False, norm='slaney') -> [n_mels, n_fft//2+1] f32."""
    fmax = sr / 2.0 if fmax is None else fmax
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0

    def hz2mel(f):
        f = np.asarray(f, dtype=np.float64)
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, f / f_sp)

    def mel2hz(m):
        m = np.asarray(m, dtype=np.float64)
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fft_f = np.linspace(0.0, sr / 2.0, n_fft // 2 + 1)
    hz = mel2hz(np.linspace(hz2mel(fmin), hz2mel(fmax), n_mels + 2))
    ramps = hz[:, None] - fft_f[None, :]
    fdiff = np.diff(hz)
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    w = np.maximum(0.0, np.minimum(lower, upper)) * (2.0 / (hz[2:] - hz[:-2]))[:, None]
    return w.astype(np.float32)


def get_bank(sr, n_fft, n_mels, fmin, fmax, device):
    key = (sr, n_fft, n_mels, fmin, fmax, str(device))
    if key not in _banks:
        _banks[key] = ops.MelBank(slaney_filterbank(sr, n_fft, n_mels, fmin, fmax), device)
    return _banks[key]


def _check(n_fft, win_size, center):
    if center:
        raise NotImplementedError("center=True on top of the manual reflect padding (a double reflection) is not a configuration "
                                  "the reference uses; ops.stft(center=True) gives torch.stft's own centred transform")
    if n_fft < 256 or n_fft > 4096 or n_fft & (n_fft - 1) or win_size > n_fft or win_size & (win_size - 1):
        raise NotImplementedError("n_fft must be a power of two in [256, 4096] and win_size a power of two <= n_fft")


def spectrogram_torch(y, n_fft, sampling_rate, hop_size, win_size, center=False, lengths=None):
    """mel_processing.py:40-74: y [B, L] -> |X| [B, n_fft//2+1, T].  lengths (optional int32 [B]): per-row valid samples."""
    _check(n_fft, win_size, center)
    bank = get_bank(sampling_rate, n_fft, 128, 0.0, None, y.device)
    spec, _ = ops.mel_frontend(y, bank, hop_size, want_spec=True, want_mel=False, lens=lengths, n_fft=n_fft, win=win_size)
    return ops.to_channels_first(spec)


def spec_to_mel_torch(spec, n_fft, num_mels, sampling_rate, fmin, fmax):
    """mel_processing.py:77-90: |X| [B, F, T] -> log-mel [B, num_mels, T]."""
    bank = get_bank(sampling_rate, n_fft, num_mels, fmin, fmax, spec.device)
    return ops.to_channels_first(ops.spec_to_mel(ops.to_channels_last(spec, pad_to=4), bank))


def mel_spectrogram_torch(y, n_fft, num_mels, sampling_rate, hop_size, win_size, fmin, fmax, center=False):
    """mel_processing.py:93-142: y [B, L] -> log-mel [B, num_mels, T]; differentiable wrt y."""
    _check(n_fft, win_size, center)
    bank = get_bank(sampling_rate, n_fft, num_mels, fmin, fmax, y.device)
    _, mel = ops.mel_frontend(y, bank, hop_size, want_spec=False, want_mel=True, n_fft=n_fft, win=win_size)
    return ops.to_channels_first(mel) if not mel.requires_grad else _CFirst.apply(mel)


class _CFirst(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return ops.to_channels_first(x)

    @staticmethod
    def backward(ctx, dy):
        return ops.to_channels_last(dy)
