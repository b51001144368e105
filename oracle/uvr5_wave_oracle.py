"""CPU restatement of SeparateVR.separate (uvr5/separate.py:103-196) from the decoded waveform to the two output waveforms,
with numpy restatements of the three librosa 0.9.2 functions it calls (librosa is not a dependency of this project):

  stft      librosa.stft(y, n_fft, hop_length) with its defaults: periodic Hann(n_fft), center=True with n_fft // 2 samples of
            padding on each side in pad_mode PAD_MODE, 1 + L // hop frames, rfft of each windowed frame in float64, stored
            as complex64 for a float32 signal
  istft     librosa.istft(stft_matrix, hop_length): n_fft = 2 (bins - 1), irfft of each frame times the window,
            overlap-add, division by the window sum-square wherever it exceeds numpy's tiny, trimming n_fft // 2 from both
            ends (hop (T - 1) samples), float64 for a complex128 input
  resample  librosa.resample(y, orig_sr, target_sr, res_type): y itself for equal rates; "polyphase" is
            scipy.signal.resample_poly(y, target / g, orig / g) with g = gcd, "scipy" is scipy.signal.resample; then
            fix_length to int(ceil(L * target / orig)) and the input dtype

PAD_MODE: librosa 0.9.0 changed stft's default pad_mode from "reflect" to "constant" (zero padding); this restatement takes
"constant" for 0.9.2 without a run of that version to confirm it.  It only affects the first and last n_fft / 2 samples of
each band.  uvr5.ZERO_PAD is the device path's copy of the same choice.

The net is oracle.uvr5_oracle (CascadedASPPNet) or oracle.uvr5_echo_oracle (CascadedNet).  cmb_spectrogram_to_wave's
np.ndarray leaves memory it never writes uninitialised (band 1's bins past crop_stop, the top band's Nyquist bin); here
it is zero, as in the device path.
"""
import math

import numpy as np
import scipy.signal

from oracle import uvr5_echo_oracle, uvr5_oracle

PAD_MODE = "constant"


def hann(n):
    """scipy.signal.get_window("hann", n, fftbins=True): the periodic Hann window"""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)


def stft(y, n_fft, hop_length, pad_mode=PAD_MODE):
    y = np.asarray(y)
    yp = np.pad(y, (n_fft // 2, n_fft // 2), mode=pad_mode)
    T = 1 + (yp.shape[-1] - n_fft) // hop_length
    idx = np.arange(n_fft)[:, None] + hop_length * np.arange(T)[None, :]
    out_dtype = np.complex64 if y.dtype == np.float32 else np.complex128
    return np.fft.rfft(hann(n_fft)[:, None] * yp[idx], axis=0).astype(out_dtype)


def istft(stft_matrix, hop_length):
    n_fft = 2 * (stft_matrix.shape[0] - 1)
    T = stft_matrix.shape[1]
    dtype = np.float32 if stft_matrix.dtype == np.complex64 else np.float64
    w = hann(n_fft)
    frames = w[:, None] * np.fft.irfft(stft_matrix, n=n_fft, axis=0)
    y = np.zeros(n_fft + hop_length * (T - 1), dtype=dtype)
    wss = np.zeros_like(y)
    for t in range(T):
        y[t * hop_length:t * hop_length + n_fft] += frames[:, t]
        wss[t * hop_length:t * hop_length + n_fft] += w ** 2
    nz = wss > np.finfo(wss.dtype).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2:-(n_fft // 2)]


def fix_length(y, size):
    n = y.shape[-1]
    if n > size:
        return y[..., :size]
    if n < size:
        return np.pad(y, [(0, 0)] * (y.ndim - 1) + [(0, size - n)])
    return y


def resample(y, orig_sr, target_sr, res_type="polyphase"):
    if orig_sr == target_sr:
        return y
    n_samples = int(np.ceil(y.shape[-1] * (float(target_sr) / orig_sr)))
    if res_type in ("scipy", "fft"):
        y_hat = scipy.signal.resample(y, n_samples, axis=-1)
    elif res_type == "polyphase":
        g = np.gcd(int(orig_sr), int(target_sr))
        y_hat = scipy.signal.resample_poly(y, int(target_sr) // g, int(orig_sr) // g, axis=-1)
    else:
        raise ValueError(f"res_type {res_type!r} is not restated here")
    return np.ascontiguousarray(fix_length(y_hat, n_samples), dtype=y.dtype)


# ---- spec_utils (lib_v5/vr_network/spec_utils.py) ------------------------------------------------------------------
def combine_spectrograms(specs, param):
    l = min(specs[i].shape[2] for i in specs)
    spec_c = np.zeros((2, param["bins"] + 1, l), dtype=np.complex64)
    offset = 0
    for d in range(1, len(param["band"]) + 1):
        bp = param["band"][d]
        h = bp["crop_stop"] - bp["crop_start"]
        spec_c[:, offset:offset + h, :l] = specs[d][:, bp["crop_start"]:bp["crop_stop"], :l]
        offset += h
    gp = 1
    for b in range(param["pre_filter_start"] + 1, param["pre_filter_stop"]):
        g = math.pow(10, -(b - param["pre_filter_start"]) * (3.5 - gp) / 20.0)
        gp = g
        spec_c[:, b, :] *= g
    return spec_c


def _lp(spec, bin_start, bin_stop):
    g = 1.0
    for b in range(bin_start, bin_stop):
        g -= 1 / (bin_stop - bin_start)
        spec[:, b, :] = g * spec[:, b, :]
    spec[:, bin_stop:, :] *= 0
    return spec


def _hp(spec, bin_start, bin_stop):
    g = 1.0
    for b in range(bin_start, bin_stop, -1):
        g -= 1 / (bin_start - bin_stop)
        spec[:, b, :] = g * spec[:, b, :]
    spec[:, 0:bin_stop + 1, :] *= 0
    return spec


def mirroring(spec_m, input_high_end, param):
    lo = param["pre_filter_start"] - 10
    mirror = np.flip(np.abs(spec_m[:, lo - input_high_end.shape[1]:lo, :]), 1)
    mirror = mirror * np.exp(1.0j * np.angle(input_high_end))
    return np.where(np.abs(input_high_end) <= np.abs(mirror), input_high_end, mirror)


def cmb_spectrogram_to_wave(spec_m, param, extra_bins_h=None, extra_bins=None):
    bands = param["band"]
    n = len(bands)
    offset = 0
    wave = None
    for d in range(1, n + 1):
        bp = bands[d]
        spec_s = np.zeros((2, bp["n_fft"] // 2 + 1, spec_m.shape[2]), dtype=complex)
        h = bp["crop_stop"] - bp["crop_start"]
        spec_s[:, bp["crop_start"]:bp["crop_stop"], :] = spec_m[:, offset:offset + h, :]
        offset += h
        if d == n:
            if extra_bins_h:
                max_bin = bp["n_fft"] // 2
                spec_s[:, max_bin - extra_bins_h:max_bin, :] = extra_bins[:, :extra_bins_h, :]
            if bp["hpf_start"] > 0:
                spec_s = _hp(spec_s, bp["hpf_start"], bp["hpf_stop"] - 1)
            wave = np.add(wave, _to_wave(spec_s, bp["hl"]))
        else:
            sr = bands[d + 1]["sr"]
            if d == 1:
                spec_s = _lp(spec_s, bp["lpf_start"], bp["lpf_stop"])
                wave = _to_wave(spec_s, bp["hl"])
                if bp["sr"] != sr:
                    raise ValueError("sinc_fastest between different rates is not restated here")
            else:
                spec_s = _hp(spec_s, bp["hpf_start"], bp["hpf_stop"] - 1)
                spec_s = _lp(spec_s, bp["lpf_start"], bp["lpf_stop"])
                wave = resample(np.add(wave, _to_wave(spec_s, bp["hl"])), bp["sr"], sr, res_type="scipy")
    return wave.T


def _to_wave(spec, hop):
    return np.asarray([istft(spec[0], hop), istft(spec[1], hop)])


# ---- SeparateVR.separate ------------------------------------------------------------------------------------------
def front_end(wave, param, high_end_process="mirroring"):
    """-> (x_spec_m [2, bins + 1, l] complex64, input_high_end_h, input_high_end) of separate.py:106-143"""
    bands = param["band"]
    n = len(bands)
    x_wave, x_spec = {}, {}
    ihe_h, ihe = None, None
    for d in range(n, 0, -1):
        bp = bands[d]
        if d == n:
            x_wave[d] = np.asarray(wave, dtype=np.float32)
            if x_wave[d].ndim == 1:
                x_wave[d] = np.asfortranarray([x_wave[d], x_wave[d]])
        else:
            x_wave[d] = resample(x_wave[d + 1], bands[d + 1]["sr"], bp["sr"], bp["res_type"])
        x_spec[d] = np.asarray([stft(x_wave[d][0], bp["n_fft"], bp["hl"]), stft(x_wave[d][1], bp["n_fft"], bp["hl"])])
        if d == n and high_end_process != "none":
            ihe_h = (bp["n_fft"] // 2 - bp["crop_stop"]) + (param["pre_filter_stop"] - param["pre_filter_start"])
            ihe = x_spec[d][:, bp["n_fft"] // 2 - ihe_h:bp["n_fft"] // 2, :]
    return combine_spectrograms(x_spec, param), ihe_h, ihe


def net_inference(P, x_spec_m, param, agg, tta, net):
    """SeparateVR.inference with the oracle net: net = ("vr", enlarge) or ("echo", None)"""
    aggressiveness = {"value": float(agg / 100), "split_bin": param["band"][1]["crop_stop"],
                      "aggr_correction": param.get("aggr_correction")}
    data = {"window_size": 512, "tta": tta}
    n_fft = 2 * param["bins"]
    if net[0] == "vr":
        return uvr5_oracle.inference(P, x_spec_m, aggressiveness, data, n_fft, net[1])
    return uvr5_echo_oracle.inference(P, x_spec_m, aggressiveness, data, n_fft)


def back_end(x_spec_m, pred, x_phase, param, ihe_h=None, ihe=None):
    """-> (wav_accompaniment, wav_vocals) of separate.py:157-187, before the int16 cast"""
    y = pred * x_phase
    v = x_spec_m - y
    outs = []
    for s in (y, v):
        if ihe is not None:
            outs.append(cmb_spectrogram_to_wave(s, param, ihe_h, mirroring(s, ihe, param)))
        else:
            outs.append(cmb_spectrogram_to_wave(s, param))
    return outs[0], outs[1]


def separate(P, wave, param, agg=10, tta=False, high_end_process="mirroring", net=("vr", False)):
    """-> (accompaniment, vocals, x_spec_m)"""
    x_spec_m, ihe_h, ihe = front_end(wave, param, high_end_process)
    pred, _, x_phase = net_inference(P, x_spec_m, param, agg, tta, net)
    acc, voc = back_end(x_spec_m, pred, x_phase, param, ihe_h, ihe)
    return acc, voc, x_spec_m


def make_clip(seed, seconds, sr=44100, mono=False, extra=137):
    """Seeded float32 clip: a few tones with vibrato and noise, L = seconds * sr + extra samples ([2, L], or [L] if mono)"""
    rs = np.random.RandomState(seed)
    L = int(seconds * sr) + extra
    t = np.arange(L) / sr
    chans = []
    for _ in range(1 if mono else 2):
        x = np.zeros(L)
        for f in (110.0, 220.0 * 1.5, 440.0, 1250.0, 3500.0, 9000.0, 15000.0):
            x += rs.uniform(0.02, 0.12) * np.sin(2 * np.pi * f * t + 3 * np.sin(2 * np.pi * rs.uniform(2, 6) * t) + rs.uniform(0, 6))
        x += 0.02 * rs.randn(L)
        chans.append(x)
    out = np.asarray(chans, dtype=np.float32)
    return out[0] if mono else out
