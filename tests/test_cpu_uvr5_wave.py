"""CPU tests of the waveform-to-waveform VR separation (uvr5.separate_wave): the oracle (oracle/uvr5_wave_oracle.py) against
the reference outputs pinned in tests/golden/uvr5_wave.pt, its librosa restatement against independent computations, the
host-side filters and gain vectors, the parameter checks, and the mixed-radix STFT core compiled for the host."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import scipy.signal
import torch

from oracle import uvr5_echo_oracle, uvr5_oracle
from oracle import uvr5_wave_oracle as W
from easevoice_trainer_b200 import uvr5

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_wave.pt"), weights_only=False)


def _params(case):
    c = GOLD[case]
    n_fft = 2 * c["param"]["bins"]
    if c["net"] == "vr":
        return uvr5_oracle.init_params(uvr5_oracle.param_spec(c["size"]), c["seed"]), ("vr", False)
    return uvr5_echo_oracle.init_params(uvr5_echo_oracle.param_spec(n_fft, c["nout"]), c["seed"]), ("echo", None)


@pytest.mark.parametrize("case", ["vr", "echo"])
def test_oracle_matches_golden(case):
    c = GOLD[case]
    P, net = _params(case)
    clip = W.make_clip(c["clip_seed"], c["seconds"], mono=c["mono"])
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    acc, voc, x = W.separate(P, clip, c["param"], c["agg"], c["tta"], "mirroring", net)
    assert acc.shape == (c["n_out"], 2) and x.shape[2] == c["l"]
    assert np.allclose(x[:, :, ::GOLD["spec_stride"]], c["x_spec_m"].numpy(), rtol=0, atol=1e-6 * np.abs(x).max())
    for k, a in (("acc", acc), ("voc", voc)):
        scale = np.abs(a).max()
        for got, want in ((a[::GOLD["wave_stride"]], c[k]), (a[:GOLD["edge"]], c[k + "_head"]), (a[-GOLD["edge"]:], c[k + "_tail"])):
            assert np.abs(got - want.numpy()).max() <= 1e-5 * scale


def test_stft_matches_torch():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(3001)
    for n_fft, hop in ((640, 80), (320, 80), (512, 160), (960, 480)):
        got = W.stft(x, n_fft, hop)
        want = torch.stft(torch.from_numpy(x), n_fft, hop, window=torch.hann_window(n_fft, periodic=True, dtype=torch.float64),
                          center=True, pad_mode="constant", return_complex=True).numpy()
        assert got.shape == want.shape == (n_fft // 2 + 1, 1 + 3001 // hop)
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_istft_inverts_stft():
    rng = np.random.default_rng(2)
    for n_fft, hop in ((640, 80), (960, 480)):
        x = rng.standard_normal(hop * 40)
        y = W.istft(W.stft(x, n_fft, hop), hop)
        assert y.shape == (hop * 40,)
        assert np.abs(y - x).max() <= 1e-10


def test_fir_taps_match_scipy():
    for up, down in ((1, 3), (1, 2), (2, 3), (3, 1)):
        m = max(up, down)
        want = scipy.signal.firwin(2 * 10 * m + 1, 1.0 / m, window=("kaiser", 5.0))
        assert np.abs(uvr5.firwin_kaiser(2 * 10 * m + 1, 1.0 / m) - want).max() <= 1e-14
    # the padded filter reproduces scipy.signal.resample_poly through the same index formula as the kernel
    rng = np.random.default_rng(3)
    x = rng.standard_normal(1001).astype(np.float32)
    for up, down in ((1, 3), (1, 2)):
        h, _, npr = uvr5.poly_filter(up, down)
        want = scipy.signal.resample_poly(x, up, down)
        n = np.arange(want.shape[0])[:, None]
        i = np.arange(x.shape[0])[None, :]
        j = (n + npr) * down - i * up
        got = np.where((j >= 0) & (j < h.shape[0]), x[None, :].astype(np.float64) * h[np.clip(j, 0, h.shape[0] - 1)], 0).sum(1)
        assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


@pytest.mark.parametrize("case", ["vr", "echo"])
def test_band_gains_match_reference_filters(case):
    param = GOLD[case]["param"]
    gains = uvr5.band_gains(param)
    n = len(param["band"])
    for d, bp in param["band"].items():
        spec = np.ones((2, bp["n_fft"] // 2 + 1, 3), dtype=complex)
        if d == n:
            spec = W._hp(spec, bp["hpf_start"], bp["hpf_stop"] - 1)
        elif d == 1:
            spec = W._lp(spec, bp["lpf_start"], bp["lpf_stop"])
        else:
            spec = W._lp(W._hp(spec, bp["hpf_start"], bp["hpf_stop"] - 1), bp["lpf_start"], bp["lpf_stop"])
        assert np.array_equal(spec[0, :, 0].real, gains[d])
    specs = {}
    for d, bp in param["band"].items():
        specs[d] = np.zeros((2, bp["n_fft"] // 2 + 1, 1), np.complex64)
        specs[d][:, bp["crop_start"]:bp["crop_stop"]] = 1
    comb = W.combine_spectrograms(specs, param)
    pre = uvr5.pre_filter_gains(param)
    covered = sum(bp["crop_stop"] - bp["crop_start"] for bp in param["band"].values())
    assert np.array_equal(comb[0, :covered, 0].real, pre[:covered])
    assert uvr5.high_end_head(param) == 101


def _bad(param, **kw):
    with pytest.raises(ValueError):
        uvr5.check_wave_param(param, **kw)


def test_param_rules():
    base = GOLD["vr"]["param"]

    def mod(f):
        p = dict(base)
        p["band"] = {b: dict(x) for b, x in base["band"].items()}
        f(p)
        return p

    uvr5.check_wave_param(base)
    uvr5.check_wave_param(base, high_end_process="none")
    for k in ("mid_side", "mid_side_b2", "reverse"):
        _bad(mod(lambda p: p.__setitem__(k, True)))
    _bad(mod(lambda p: p["band"][3].__setitem__("sr", 14000)))                 # 44100 / 14000 is not an integer
    _bad(mod(lambda p: p["band"][3].__setitem__("res_type", "kaiser_fast")))
    _bad(mod(lambda p: p["band"][1].__setitem__("sr", 3675)))                  # sinc_fastest between 3675 and 7350 Hz
    _bad(mod(lambda p: p["band"][1].__setitem__("n_fft", 1344)))               # 1344 = 2^6 3 7
    _bad(mod(lambda p: p["band"][4].__setitem__("n_fft", 15360)))              # above the core's limit
    _bad(mod(lambda p: p.__setitem__("sr", 48000)))
    _bad(base, high_end_process="mirroring2")
    _bad(base, high_end_process="bypass")


def test_short_input_raises():
    class _M:
        output_bin = 673
    with pytest.raises(ValueError):
        uvr5.separate_wave(np.zeros((2, 400), np.float32), _M(), GOLD["vr"]["param"])


def test_lengths_match_librosa():
    param = GOLD["vr"]["param"]
    lens = uvr5.band_lengths(GOLD["vr"]["clip_len"], param)
    x = np.zeros((2, GOLD["vr"]["clip_len"]), np.float32)
    for d in (3, 2, 1):
        x = W.resample(x, param["band"][d + 1]["sr"], param["band"][d]["sr"], "polyphase")
        assert x.shape[1] == lens[d]


# ---- the mixed-radix core on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("stft_mr") / "libstft_mr_host.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tools", "exp", "stft_mr_host_test.cpp")], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("N", [320, 640, 960, 480, 1536, 256, 512, 1024, 2048, 4096])
def test_mixed_radix_core_matches_numpy(host_lib, N):
    assert host_lib.stft_mr_size_supported(N) == 1
    rng = np.random.default_rng(N)
    L = 9000
    wav = (rng.random(L) - 0.5).astype(np.float32)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)
    for s0 in (-N // 2, 1000, L - N // 2 - 1):                   # left edge, interior, right edge
        for zero_pad in (0, 1):
            X = np.zeros((N // 2 + 1) * 2, np.float32)
            host_lib.stft_mr_frame_fwd(_p(wav), L, s0, N, zero_pad, 256, _p(X))
            idx = s0 + np.arange(N)
            if zero_pad:
                seg = np.where((idx >= 0) & (idx < L), wav[np.clip(idx, 0, L - 1)], 0).astype(np.float64)
            else:
                i = np.abs(idx)
                seg = wav[np.where(i >= L, 2 * (L - 1) - i, i)].astype(np.float64)
            ref = np.fft.rfft(seg * w)
            got = X[0::2] + 1j * X[1::2]
            assert np.abs(got - ref).max() / np.abs(ref).max() < 2e-6
    G = rng.standard_normal((N // 2 + 1) * 2).astype(np.float32)
    S = np.zeros(N, np.float32)
    host_lib.stft_mr_frame_adj(_p(G), N, 256, _p(S))
    Gc = G[0::2] + 1j * G[1::2]
    k, n = np.arange(N // 2 + 1)[:, None], np.arange(N)[None, :]
    Sref = (Gc[:, None] * np.exp(2j * np.pi * k * n / N)).real.sum(0)
    assert np.abs(S - Sref).max() / np.abs(Sref).max() < 2e-6


def test_unsupported_sizes(host_lib):
    for N in (1344, 1152, 15, 8, 7681, 15360):
        assert host_lib.stft_mr_size_supported(N) == 0
        assert not uvr5.stft_size_ok(N)
