"""CPU restatement of `Normalize._name2go` (reference src/normalization/normalize.py:151-179), the per-file body of
`Normalize.ssl`, in numpy / float64, plus a literal restatement of the resampler that librosa 0.9.2 calls there.

TEST INFRASTRUCTURE ONLY (tests/, oracle/pin_normalize_ssl.py, the CPU arm of tools/bench_normalize_ssl.py).  Imports nothing
from the product.

  skip / status   normalize.py:153-158   m = np.abs(a).max(); m > 2.2 (a float32 scalar against a Python float: float64)
  normalisation   normalize.py:159-160   float32 operations in the reference's order, constants rounded to float32
  resampling      normalize.py:161-163   librosa.resample(..., 32000, 16000), res_type kaiser_best = resampy, fix=True
  model           normalize.py:166-168   oracle/hubert_oracle.forward
  NaN check       normalize.py:169-170
  outputs         normalize.py:172-178   int16 waveform (x86 astype: truncate to int32, keep 16 bits), [1, 768, T] features

Resampling: resampy's `sinc_window` (filters.py) and `resample_f` (interpn.py) are restated literally below
(`sinc_window_literal`, `resample_f_literal`); with sample_ratio = 1/2 the loop reads the table at offsets 0 and 1/2 only,
which `resample_taps` states in closed form.  tests/test_cpu_normalize_ssl.py checks that the two agree.
"""
import numpy as np
import scipy.signal
import torch

from oracle import hubert_oracle

MAXX, ALPHA = 0.95, 0.5                                   # normalize.py:62-63
# resampy kaiser_best (the filter librosa 0.9.2's default res_type names)
KAISER_BEST = dict(num_zeros=64, precision=16, rolloff=0.9475937167399596, beta=14.769656459379492)
OK, SKIP, NONFINITE = "ok", "skip", "nonfinite"


def normalize(a):
    """normalize.py:155-160 on float32 samples a -> (status, a32 float32, a32b float32).  status SKIP: m > 2.2; NONFINITE: the
    outputs are NaN (m == 0 or a NaN sample), which makes the model output NaN and the reference write nothing."""
    a = np.asarray(a, dtype=np.float32)
    m = np.abs(a).max()                                          # raises on an empty array, as in the reference
    if float(m) > 2.2:
        return SKIP, None, None
    with np.errstate(invalid="ignore", divide="ignore"):
        a32 = (a / m * np.float32(MAXX * ALPHA * 32768)) + np.float32((1 - ALPHA) * 32768) * a
        a32b = (a / m * np.float32(MAXX * ALPHA * 1145.14)) + np.float32((1 - ALPHA) * 1145.14) * a
    return (NONFINITE if not m > 0 else OK), a32, a32b


def to_int16(a32):
    """`a32.astype("int16")` as numpy does it on x86-64: C float -> int32 truncation (cvttss2si), low 16 bits kept"""
    return a32.astype(np.int32).astype(np.int16)


def resample_taps(num_zeros=64, precision=16, rolloff=KAISER_BEST["rolloff"], beta=KAISER_BEST["beta"]):
    """The table entries resample_f reads at ratio 1/2, already scaled by the ratio: h[j] = 0.5 * win[j * 2^precision / 2],
    win = rolloff sinc(rolloff x) kaiser, for j = 0 .. 2 num_zeros - 1."""
    n2 = 2 * num_zeros
    j = np.arange(n2, dtype=np.float64)
    return 0.5 * rolloff * np.sinc(rolloff * j / 2) * np.i0(beta * np.sqrt(1.0 - (j / n2) ** 2)) / np.i0(beta)


def resample(y):
    """librosa.resample(y, orig_sr=32000, target_sr=16000) with its 0.9.2 defaults, closed form, float64 sums:
    y16[n] = sum_{|d| < 128} h[|d|] y[2n + d] for n < floor(L / 2), then one zero for odd L (fix_length to ceil(L / 2));
    the result is cast back to y's dtype (float32) like librosa."""
    y = np.asarray(y)
    h = resample_taps()
    L = y.shape[-1]
    x = np.concatenate([np.zeros(127), y.astype(np.float64), np.zeros(127)])
    n = L // 2
    out = np.zeros((L + 1) // 2, dtype=np.float64)
    for d in range(-127, 128):
        out[:n] += h[abs(d)] * x[127 + d:127 + d + 2 * n:2]
    return out.astype(y.dtype)


def sinc_window_literal(num_zeros=64, precision=16, rolloff=KAISER_BEST["rolloff"], beta=KAISER_BEST["beta"]):
    """resampy.filters.sinc_window with window = scipy.signal.kaiser(beta): the right wing of the interpolation table"""
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = scipy.signal.windows.kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win, num_bits


def resample_f_literal(x, sample_ratio, interp_win, num_table):
    """resampy.interpn.resample_f for one channel, the loop as written (float64 output instead of x's dtype), after
    resampy.resample's `interp_win *= sample_ratio` and int(L * ratio) outputs"""
    interp_win = interp_win * sample_ratio
    interp_delta = np.zeros_like(interp_win)
    interp_delta[:-1] = np.diff(interp_win)
    y = np.zeros(int(x.shape[0] * sample_ratio), dtype=np.float64)
    scale = min(1.0, sample_ratio)
    time_increment = 1.0 / sample_ratio
    index_step = int(scale * num_table)
    time_register = 0.0
    nwin = interp_win.shape[0]
    n_orig = x.shape[0]
    for t in range(y.shape[0]):
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        i_max = min(n + 1, (nwin - offset) // index_step)
        for i in range(i_max):
            weight = interp_win[offset + i * index_step] + eta * interp_delta[offset + i * index_step]
            y[t] += weight * x[n - i]
        frac = scale - frac
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
        for k in range(k_max):
            weight = interp_win[offset + k * index_step] + eta * interp_delta[offset + k * index_step]
            y[t] += weight * x[n + k + 1]
        time_register += time_increment
    return y


def librosa_resample_literal(y, win=None):
    """librosa 0.9.2 resample(y, 32000, 16000) through the literal resampy loop: resampy, then fix_length to ceil(L / 2)"""
    interp_win, num_table = win if win is not None else sinc_window_literal()
    y16 = resample_f_literal(np.asarray(y, dtype=np.float64), 0.5, interp_win, num_table)
    return np.concatenate([y16, np.zeros(-(-len(y) // 2) - len(y16))])


def name2go(a, P, m):
    """normalize.py:151-179 for samples a with HuBERT weights P (config m) -> dict(status, wav int16 or None, ssl [1, 768, T]
    float32 or None); status NONFINITE also covers NaN features (normalize.py:169-170)."""
    status, a32, a32b = normalize(a)
    if status == SKIP:
        return dict(status=SKIP, wav=None, ssl=None)
    a16 = resample(a32b)
    with torch.no_grad():
        ssl = hubert_oracle.forward(P, torch.from_numpy(a16)[None], m).transpose(1, 2)
    if bool(torch.isnan(ssl).any()):
        return dict(status=NONFINITE, wav=None, ssl=None)
    return dict(status=OK, wav=to_int16(a32), ssl=ssl.detach().contiguous())


def clip(spec):
    """The seeded test clips of tests/golden/normalize_ssl.pt: spec = dict(n, seed, peak) -> float32 [n]: white noise scaled so
    that max |a| == peak (peak 0: silence)."""
    if spec["peak"] == 0:
        return np.zeros(spec["n"], dtype=np.float32)
    x = torch.randn(spec["n"], generator=torch.Generator().manual_seed(spec["seed"])).numpy().astype(np.float32)
    return (x * np.float32(spec["peak"] / np.abs(x).max())).astype(np.float32)
