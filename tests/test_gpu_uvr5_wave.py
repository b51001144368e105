"""GPU tests of the waveform-to-waveform VR separation (`pytest -m gpu`): the band STFT, iSTFT at the mixed-radix sizes,
polyphase and FFT resampling, and the spectrum assembly against float64 / scipy / the oracle, then uvr5.separate_wave
against the reference outputs pinned in tests/golden/uvr5_wave.pt (oracle/pin_uvr5_wave.py)."""
import os

import numpy as np
import pytest
import scipy.signal
import torch

from oracle import uvr5_echo_oracle, uvr5_oracle
from oracle import uvr5_wave_oracle as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "uvr5_wave.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
BANDS = ((640, 80), (320, 80), (512, 160), (960, 480))


@pytest.fixture(scope="module")
def mods():
    from easevoice_trainer_b200 import lib, ops, uvr5
    lib.init().evk_set_precise(0)
    return ops, uvr5


def _precise(on):
    from easevoice_trainer_b200 import lib
    lib.init().evk_set_precise(1 if on else 0)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_band_stft_vs_float64(mods):
    ops, _ = mods
    rng = np.random.default_rng(5)
    wavs = [rng.standard_normal((2, 3001 + 7 * i)).astype(np.float32) for i in range(4)]
    buf = torch.from_numpy(np.concatenate([w.ravel() for w in wavs])).to(DEV)
    l = min(1 + w.shape[1] // hop for w, (_, hop) in zip(wavs, BANDS))
    bands, off, row0 = [], 0, 0
    for w, (n, hop) in zip(wavs, BANDS):
        bands.append((off, w.shape[1], w.shape[1], n, hop, 0, n // 2 + 1, row0))
        off, row0 = off + w.size, row0 + n // 2 + 1
    spec, high = ops.vr_band_stft(buf, bands, l, torch.ones(row0, device=DEV), row0, high_band=3, high_lo=379, high_h=101)
    got = torch.view_as_complex(spec).cpu().numpy()
    row0 = 0
    for w, (n, hop) in zip(wavs, BANDS):
        want = np.stack([W.stft(w[c].astype(np.float64), n, hop)[:, :l] for c in range(2)])
        g = got[:, row0:row0 + n // 2 + 1]
        assert np.abs(g - want).max() <= 2e-6 * np.abs(want).max(), (n, hop)
        row0 += n // 2 + 1
    assert np.array_equal(torch.view_as_complex(high).cpu().numpy(), got[:, row0 - 481 + 379:row0 - 481 + 480])


@pytest.mark.parametrize("n,hop", BANDS)
def test_istft_mixed_sizes_vs_float64(mods, n, hop):
    ops, _ = mods
    rng = np.random.default_rng(n)
    X = (rng.standard_normal((4, 50, n // 2 + 1)) + 1j * rng.standard_normal((4, 50, n // 2 + 1)))
    got = ops.istft(torch.view_as_real(torch.from_numpy(X.astype(np.complex64))).contiguous().to(DEV), 4, 1, n, hop).cpu().numpy()
    want = np.stack([W.istft(X[r].T, hop) for r in range(4)])
    assert np.abs(got - want).max() <= 5e-6 * np.abs(want).max()


@pytest.mark.parametrize("up,down", [(1, 3), (1, 2)])
def test_resample_poly_vs_scipy(mods, up, down):
    ops, uvr5 = mods
    x = np.random.default_rng(up + down).standard_normal((2, 10007)).astype(np.float32)
    h, _, npr = uvr5.poly_filter(up, down)
    want = scipy.signal.resample_poly(x, up, down, axis=-1)
    got = ops.resample_poly(torch.from_numpy(x).to(DEV), torch.from_numpy(h).to(DEV), up, down, npr, want.shape[1]).cpu().numpy()
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def test_fft_resample_vs_scipy(mods):
    _, uvr5 = mods
    x = np.random.default_rng(9).standard_normal((4, 80 * 367))
    for ratio in (2, 3):
        want = scipy.signal.resample(x, x.shape[1] * ratio, axis=-1)
        got = uvr5.fft_resample(torch.from_numpy(x).to(DEV), x.shape[1] * ratio).cpu().numpy()
        assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def test_assembly_vs_oracle(mods):
    ops, uvr5 = mods
    param = GOLD["vr"]["param"]
    rng = np.random.default_rng(11)
    l, rows = 20, param["bins"] + 1
    x = ((rng.standard_normal((2, rows, l)) + 1j * rng.standard_normal((2, rows, l))) * 0.3).astype(np.complex64)
    x[:, 5, 3] = 0                                                   # a zero bin: phase 1
    pred = rng.random((2, rows, l)).astype(np.float32)
    hh = uvr5.high_end_head(param)
    ihe = ((rng.standard_normal((2, hh, l)) + 1j * rng.standard_normal((2, hh, l))) * 0.2).astype(np.complex64)
    coef = np.float32(1.7)
    bands, row0 = [], 0
    for d in range(1, 5):
        bp = param["band"][d]
        bands.append((bp["n_fft"], bp["crop_start"], bp["crop_stop"], row0))
        row0 += bp["crop_stop"] - bp["crop_start"]
    gains = [torch.from_numpy(g.astype(np.float32)).to(DEV) for g in uvr5.band_gains(param).values()]
    dx = torch.view_as_real(torch.from_numpy(x)).contiguous().to(DEV)
    frames = ops.vr_assemble(dx, torch.from_numpy(pred).to(DEV), None, torch.tensor([coef], device=DEV), bands, gains,
                             high=torch.view_as_real(torch.from_numpy(ihe)).contiguous().to(DEV),
                             mirror_lo=param["pre_filter_start"] - 10 - hh, top=3)
    p = pred * coef
    y = p * np.exp(1.0j * np.angle(x))
    for sig, s in enumerate((y, x - y)):
        mir = W.mirroring(s, ihe, param)
        off = 0
        for d in range(1, 5):
            bp = param["band"][d]
            spec = np.zeros((2, bp["n_fft"] // 2 + 1, l), complex)
            h = bp["crop_stop"] - bp["crop_start"]
            spec[:, bp["crop_start"]:bp["crop_stop"]] = s[:, off:off + h]
            off += h
            if d == 4:
                spec[:, 480 - hh:480] = mir
                spec = W._hp(spec, bp["hpf_start"], bp["hpf_stop"] - 1)
            elif d == 1:
                spec = W._lp(spec, bp["lpf_start"], bp["lpf_stop"])
            else:
                spec = W._lp(W._hp(spec, bp["hpf_start"], bp["hpf_stop"] - 1), bp["lpf_start"], bp["lpf_stop"])
            got = torch.view_as_complex(frames[d - 1]).cpu().numpy()[2 * sig:2 * sig + 2].transpose(0, 2, 1)
            assert np.abs(got - spec).max() <= 1e-6 * np.abs(spec).max(), (sig, d)


def _model(uvr5, case):
    c = GOLD[case]
    n_fft = 2 * c["param"]["bins"]
    if c["net"] == "vr":
        P = uvr5_oracle.init_params(uvr5_oracle.param_spec(c["size"]), c["seed"])
        return uvr5.CascadedASPPNet(n_fft, c["size"]).to(DEV).load_state_dict(P)
    P = uvr5_echo_oracle.init_params(uvr5_echo_oracle.param_spec(n_fft, c["nout"]), c["seed"])
    return uvr5.CascadedNet(n_fft, c["nout"]).to(DEV).load_state_dict(P)


def _clip(case):
    c = GOLD[case]
    return W.make_clip(c["clip_seed"], c["seconds"], mono=c["mono"])


def test_front_end_vs_golden(mods):
    ops, uvr5 = mods
    c = GOLD["vr"]
    param, clip = c["param"], _clip("vr")
    lens = uvr5.band_lengths(clip.shape[1], param)
    waves = {4: clip}
    for d in (3, 2, 1):
        waves[d] = W.resample(waves[d + 1], param["band"][d + 1]["sr"], param["band"][d]["sr"], "polyphase")
    buf = torch.from_numpy(np.concatenate([waves[d].ravel() for d in (1, 2, 3, 4)])).to(DEV)
    bands, off, row0 = [], 0, 0
    for d in (1, 2, 3, 4):
        bp = param["band"][d]
        bands.append((off, lens[d], lens[d], bp["n_fft"], bp["hl"], bp["crop_start"], bp["crop_stop"], row0))
        off, row0 = off + 2 * lens[d], row0 + bp["crop_stop"] - bp["crop_start"]
    spec, _ = ops.vr_band_stft(buf, bands, c["l"], torch.from_numpy(uvr5.pre_filter_gains(param)).to(DEV), param["bins"] + 1)
    got = torch.view_as_complex(spec).cpu().numpy()[:, :, ::GOLD["spec_stride"]]
    want = c["x_spec_m"].numpy()
    assert np.linalg.norm(got - want) / np.linalg.norm(want) <= 1e-5


def _check(c, acc, voc, tol):
    assert acc.shape == voc.shape == (c["n_out"], 2) and acc.dtype == np.float32
    for k, a in (("acc", acc), ("voc", voc)):
        assert rel(a[::GOLD["wave_stride"]], c[k]) <= tol, k
        assert rel(a[:GOLD["edge"]], c[k + "_head"]) <= tol and rel(a[-GOLD["edge"]:], c[k + "_tail"]) <= tol, k


@pytest.mark.parametrize("case", ["vr", "echo"])
def test_separate_wave_vs_golden(mods, case):
    _, uvr5 = mods
    c = GOLD[case]
    model = _model(uvr5, case)
    clip = _clip(case)
    acc, voc = uvr5.separate_wave(clip, model, c["param"], c["agg"], c["tta"])
    _check(c, acc, voc, 1e-3)
    acc2, voc2 = uvr5.separate_wave(clip, model, c["param"], c["agg"], c["tta"], max_windows=1)
    assert np.array_equal(acc, acc2) and np.array_equal(voc, voc2)                # batching does not change a bit
    acc3, voc3 = uvr5.separate_wave(clip, model, c["param"], c["agg"], c["tta"])
    assert np.array_equal(acc, acc3) and np.array_equal(voc, voc3)                # reproducible
    if c["mono"]:
        acc4, voc4 = uvr5.separate_wave(np.stack([clip, clip]), model, c["param"], c["agg"], c["tta"])
        assert np.array_equal(acc, acc4) and np.array_equal(voc, voc4)
    _precise(True)
    try:
        acc, voc = uvr5.separate_wave(clip, model, c["param"], c["agg"], c["tta"])
    finally:
        _precise(False)
    _check(c, acc, voc, 1e-5)


def test_all_zero_input_is_nan(mods):
    _, uvr5 = mods
    c = GOLD["vr"]
    acc, voc = uvr5.separate_wave(np.zeros((2, 48000), np.float32), _model(uvr5, "vr"), c["param"])
    assert np.isnan(acc).all() and np.isnan(voc).all()
