"""CPU rehearsal of tests/spectral_ref.py.  The general kernels' frame transforms run on the host through the real stft_core.cuh
(tools/exp/stft_host_test.cpp, stft_mr_host_test.cpp), built twice: without FMA contraction and with -mfma -ffp-contract=fast,
the two forms of the complex multiply the model covers.  The warp kernel's 32 x 32 register FFT and untangle are restated in
numpy fp32 (fmaf as a float64 product-sum rounded once), and the magnitude, filterbank, log, adjoint, overlap-add and
inverse-STFT stages in fp32 in the kernels' order.  Every emulation stays within the model at every element, for every
transform size the GPU tests use, and each modelled fault leaves the gate on at least one element."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from easevoice_trainer_b200.mel_processing import slaney_filterbank
from tests import cudacore_ref as R
from tests import spectral_ref as S
from tests.test_cpu_cudacore_ref import outside, within_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
HAS_FMA = os.path.exists("/proc/cpuinfo") and " fma" in open("/proc/cpuinfo").read()
FLAGS = {"plain": ["-ffp-contract=off"], "fma": ["-mfma", "-ffp-contract=fast"]}


def _build(tmp, src, flags):
    so = str(tmp / (os.path.basename(src).replace(".cpp", "") + "_" + "_".join(f.strip("-") for f in flags) + ".so"))
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", *flags, "-o", so, os.path.join(ROOT, "tools", "exp", src)], check=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module", params=["plain", "fma"])
def host(request, tmp_path_factory):
    if request.param == "fma" and not HAS_FMA:
        pytest.skip("this CPU has no FMA unit")
    tmp = tmp_path_factory.mktemp("spectral_" + request.param)
    pw2 = _build(tmp, "stft_host_test.cpp", FLAGS[request.param])
    mr = _build(tmp, "stft_mr_host_test.cpp", FLAGS[request.param])
    yield pw2, mr
    pw2.stft_set_fault(-1, 0)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def pow2(N):
    return N & (N - 1) == 0


# ---- fp32 emulation of the kernels ------------------------------------------------------------------------------------------
def frame_fwd(host, wav, L, s0, N, win):
    """X [N/2+1] complex (fp32 parts) of the frame at s0 through the host build of stft_core.cuh"""
    X = np.zeros((N // 2 + 1) * 2, f32)
    if pow2(N):
        host[0].stft_frame_fwd(_p(wav), L, s0, N, win, 256, _p(X))
    else:
        assert win == N
        host[1].stft_mr_frame_fwd(_p(wav), L, s0, N, 0, 256, _p(X))
    return X[0::2].astype(np.float64) + 1j * X[1::2]


def frame_adj(host, G, N):
    """S[n] = sum_k Re(G_k e^{+2 pi i k n / N}) in fp32 through the host build; G complex [N/2+1]"""
    g = np.stack([G.real, G.imag], -1).astype(f32).reshape(-1)
    out = np.zeros(N, f32)
    (host[0].stft_frame_adj if pow2(N) else host[1].stft_mr_frame_adj)(_p(g), N, 256, _p(out))
    return out


def hann_f32(N, win):
    """the kernels' fp32 window: the table entry of Hann(win) centred in the frame"""
    tab = S.TAB if pow2(N) else S.TAB_MR
    j = np.arange(N) - (N - win) // 2
    h = (0.5 - 0.5 * np.cos(2 * np.pi * (j % win) * (tab // win) / tab)).astype(f32)
    return np.where((j >= 0) & (j < win), h, f32(0))


def fmaf(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def brev5(k):
    return int(f"{k:05b}"[::-1], 2)


C32 = np.cos(2 * np.pi * np.arange(16) / 32).astype(f32)
S32 = np.sin(2 * np.pi * np.arange(16) / 32).astype(f32)


def fft32(xr, xi):
    """mel.cu fft32_regs over axis 0 (32 registers) of [32, lanes] fp32: DIF, X[k] in element brev5(k)"""
    xr, xi = xr.copy(), xi.copy()
    half = 16
    while half >= 1:
        for blk in range(0, 32, 2 * half):
            for j in range(half):
                i0, i1, tw = blk + j, blk + j + half, j * (16 // half)
                ar, ai, br, bi = xr[i0].copy(), xi[i0].copy(), xr[i1].copy(), xi[i1].copy()
                xr[i0], xi[i0] = ar + br, ai + bi
                dr, di = ar - br, ai - bi
                if tw == 0:
                    xr[i1], xi[i1] = dr, di
                elif tw == 8:
                    xr[i1], xi[i1] = di, -dr
                else:
                    xr[i1] = fmaf(dr, C32[tw], (di * S32[tw]).astype(f32))
                    xi[i1] = fmaf(di, C32[tw], (-dr * S32[tw]).astype(f32))
        half //= 2
    return xr, xi


def cmul(ar, ai, br, bi):
    return (ar * br).astype(f32) - (ai * bi).astype(f32), (ar * bi).astype(f32) + (ai * br).astype(f32)


def warp_frame_fwd(frame):
    """mel.cu mel_fwd_warp_kernel's transform of one 2048-sample frame (fp32): X [1025] complex"""
    tw = np.exp(-2j * np.pi * np.arange(2048) / 2048)
    twr, twi = tw.real.astype(f32), tw.imag.astype(f32)
    h = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(2048) / 2048)).astype(f32)
    a = (frame.astype(f32) * h).astype(f32)
    m = np.arange(1024).reshape(32, 32)                                         # m = 32 n1 + t: [n1, t]
    xr, xi = fft32(a[2 * m], a[2 * m + 1])
    k1 = np.arange(32)
    t32 = np.exp(-2j * np.pi * ((np.arange(32)[None, :] * k1[:, None]) % 1024) / 1024)
    A_r, A_i = xr[[brev5(k) for k in k1]], xi[[brev5(k) for k in k1]]         # [k1, t]
    zr, zi = cmul(A_r, A_i, t32.real.astype(f32), t32.imag.astype(f32))
    yr, yi = fft32(zr.T.copy(), zi.T.copy())                                   # lane t owns k1 = t: registers n2 = former t
    Zr, Zi = np.zeros(1024, f32), np.zeros(1024, f32)
    for k2 in range(32):
        Zr[np.arange(32) + 32 * k2], Zi[np.arange(32) + 32 * k2] = yr[brev5(k2)], yi[brev5(k2)]
    k = np.arange(1025)
    zkr, zki = Zr[k % 1024], Zi[k % 1024]
    zcr, zci = Zr[(1024 - k) & 1023], -Zi[(1024 - k) & 1023]
    sr, si = (f32(0.5) * (zkr + zcr)).astype(f32), (f32(0.5) * (zki + zci)).astype(f32)
    dr, di = (f32(0.5) * (zkr - zcr)).astype(f32), (f32(0.5) * (zki - zci)).astype(f32)
    tr, ti = cmul(twr[k], twi[k], dr, di)
    return (sr + ti).astype(np.float64) + 1j * (si - tr).astype(np.float64)


def magnitude_f32(X, eps=S.EPS):
    re, im = X.real.astype(f32), X.imag.astype(f32)
    return np.sqrt(((re * re).astype(f32) + (im * im).astype(f32)).astype(f32) + f32(eps)).astype(f32)


def csr(fb):
    ptr, idx, val = [0], [], []
    for m in range(fb.shape[0]):
        nz = np.nonzero(fb[m])[0]
        idx += nz.tolist(); val += fb[m, nz].tolist()
        ptr.append(len(idx))
    return np.array(ptr), np.array(idx), np.array(val, f32)


def mel_f32(spec, fb, shift=0):
    """[F, nb] |X| -> acc [F, n_mels] by the CSR fmaf chain (shift: every column read one bin off) and logf(fmaxf(acc, clip))"""
    ptr, idx, val = csr(fb)
    acc = np.zeros((spec.shape[0], fb.shape[0]), f32)
    for m in range(fb.shape[0]):
        for e in range(ptr[m], ptr[m + 1]):
            acc[:, m] = fmaf(val[e], spec[:, min(idx[e] + shift, spec.shape[1] - 1)], acc[:, m])
    return np.log(np.maximum(acc, f32(S.CLIP))).astype(f32)


def mel_bwd_G_f32(dmel, lm, X, fb, ge=False):
    """stft_bwd_kernel's log-mel path per frame: g_m, dmag in mel order, G = dmag / |X| * X (ge: `>=` in the clip test)"""
    lclip = np.log(f32(S.CLIP)).astype(f32)
    live = (lm >= lclip) if ge else (lm > lclip)
    gm = np.where(live, (dmel * np.exp(-lm).astype(f32)).astype(f32), f32(0))
    ptr, idx, val = csr(fb)
    dmag = np.zeros((X.shape[0], X.shape[1]), f32)
    for m in range(fb.shape[0]):
        for e in range(ptr[m], ptr[m + 1]):
            dmag[:, idx[e]] = (dmag[:, idx[e]] + (val[e] * gm[:, m]).astype(f32)).astype(f32)
    s = (dmag / magnitude_f32(X)).astype(f32)
    return (s * X.real.astype(f32)).astype(f32) + 1j * (s * X.imag.astype(f32)).astype(f32)


def ola_f32(fr, Lrow, N, hop, pad, Tr, base, skip=None):
    """stft_ola_kernel: candidates n, -n, 2 (Lrow - 1) - n, frames ascending, fp32, then dwav += acc (skip: a frame left out)"""
    n = np.arange(Lrow)
    acc = np.zeros(Lrow, f32)
    for ci, s in enumerate((n, -n, 2 * (Lrow - 1) - n)):
        r = np.abs(s)
        r = np.where(r >= Lrow, 2 * (Lrow - 1) - r, r)
        ok = (r == n) & ~((ci == 1) & (n == 0)) & ~((ci == 2) & (s == n))
        for f in range(Tr):
            j = s - f * hop + pad
            use = ok & (j >= 0) & (j < N) & (f != skip)
            acc[use] = (acc[use] + fr[f, j[use]]).astype(f32)
    out = base.copy()
    out[:Lrow] = (out[:Lrow] + acc).astype(f32)
    return out


def reflect(i, L):
    i = np.abs(i)
    return np.where(i >= L, 2 * (L - 1) - i, i)


# ---- reference helpers --------------------------------------------------------------------------------------------------------
def ref_X(wav, N, win, s0s, warp=False):
    """float64 X and its bound E (re and im stacked) of frames starting at s0s of a reflect-padded row"""
    L = wav.shape[0]
    w = S.window(N, win).numpy()
    idx = reflect(np.asarray(s0s)[:, None] + np.arange(N)[None, :], L)
    a = wav.astype(np.float64)[idx] * w
    X = np.fft.rfft(a, axis=-1)
    e = S.c_forward(N, warp) * R.U32 * np.abs(a).sum(-1)
    return X, torch.tensor(e)[:, None].expand(-1, N // 2 + 1)


def as_E(X, e):
    return R.E(torch.view_as_real(torch.as_tensor(X)), torch.stack([e, e], -1))


def cplx_t(X):
    return torch.view_as_real(torch.as_tensor(X))


SIZES = [(N, w) for N in (256, 512, 1024, 2048, 4096) for w in sorted({N, N // 2, 256})] + [(N, N) for N in (320, 640, 960)]


def row(seed, L, kind="noise"):
    g = np.random.default_rng(seed)
    if kind == "dc":
        return (1.0 + 0.1 * (g.random(L) - 0.5)).astype(f32)
    return (g.random(L) - 0.5).astype(f32)


@pytest.mark.parametrize("N,win", SIZES, ids=[f"N{n}-win{w}" for n, w in SIZES])
def test_frame_transforms_within_model(host, N, win):
    L = 3 * N + 37
    worst = 0.0
    for kind in ("noise", "dc"):
        wav = row(N + win, L, kind)
        s0s = [-N // 2, N // 3, L - N + N // 2 - 1]                        # left reflection, interior, right reflection
        X = np.stack([frame_fwd(host, wav, L, s, N, win) for s in s0s])
        Xr, e = ref_X(wav, N, win, s0s)
        worst = max(worst, within_model(cplx_t(X), as_E(Xr, e), f"X N={N} win={win} {kind}"))
    rng = np.random.default_rng(N)
    G = rng.standard_normal(N // 2 + 1) + 1j * rng.standard_normal(N // 2 + 1)
    G = (G.real.astype(f32) + 1j * G.imag.astype(f32))
    h = hann_f32(N, win)
    got = (frame_adj(host, G, N) * h).astype(f32)
    Gt = torch.as_tensor(G)[None]
    fr, efr = S.inverse_frames(Gt, torch.zeros(1, N // 2 + 1, dtype=torch.float64), N, win)
    worst = max(worst, within_model(torch.as_tensor(got)[None], R.E(fr, efr), f"adjoint N={N} win={win}"))
    print(f"N={N} win={win}: worst err / model {worst * R.SAFETY:.3f}")


def test_warp_transform_within_model():
    L = 9000
    for kind in ("noise", "dc"):
        wav = row(7, L, kind)
        s0s = [-704, 1000, L - 2048 + 704]
        X = np.stack([warp_frame_fwd(wav[reflect(s + np.arange(2048), L)]) for s in s0s])
        Xr, e = ref_X(wav, 2048, 2048, s0s, warp=True)
        w = within_model(cplx_t(X), as_E(Xr, e), f"warp X {kind}")
        print(f"warp 32 x 32: worst err / model {w * R.SAFETY:.3f}")


# ---- the whole front end and its adjoint ---------------------------------------------------------------------------------------
GEO = dict(N=1024, hop=160, win=512, sr=22050, n_mels=80)


def pipeline(host, wav, fb, dmel, base, geo=GEO, fault=None):
    """fp32 emulation of evk_stft_fwd (spec, log-mel) and evk_stft_bwd (log-mel path) on one row: (spec, mel, dwav)"""
    N, hop, win = geo["N"], geo["hop"], geo["win"]
    pad, L = (N - hop) // 2, wav.shape[0]
    T = S.frames_of_row(L, pad, N, hop)
    off = 1 if fault == "frame start" else 0
    X = np.stack([frame_fwd(host, wav, L, f * hop - pad + off, N, win) for f in range(T)])
    spec = magnitude_f32(X, 0.0 if fault == "eps" else S.EPS)
    lm = mel_f32(spec, fb, 1 if fault == "fb shift" else 0)
    G = mel_bwd_G_f32(dmel, lm, X, fb, ge=fault == "clip >=")
    if fault == "hermitian":
        G[:, 1:-1] *= 2
    h = hann_f32(N, win)
    fr = np.stack([(frame_adj(host, G[f], N) * h).astype(f32) for f in range(T)])
    return spec, lm, ola_f32(fr, L, N, hop, pad, T, base, skip=1 if fault == "ola frame" else None)


def reference(wav, fb, dmel, base, geo=GEO):
    N, hop, win = geo["N"], geo["hop"], geo["win"]
    pad, L = (N - hop) // 2, wav.shape[0]
    T = S.frames_of_row(L, pad, N, hop)
    fbt = torch.as_tensor(fb)
    x = torch.tensor(wav, dtype=torch.float64, requires_grad=True)
    X, A, counts = S.stft(x[None], None, N, hop, win, pad, T)
    mel = S.logmel_value(S.magnitude(X), fbt)
    (mel * torch.as_tensor(dmel)[None].double()).sum().backward()
    Xd = X.detach()
    spec = S.spec_E(Xd, A, N)
    lm = S.log_clip(S.mel_sum(spec, fbt))
    G, e_G = S.mel_adjoint_G(Xd, A, N, fbt, torch.as_tensor(dmel)[None].double())
    fr, efr = S.inverse_frames(G, e_G, N, win)
    dw = S.ola(fr, efr, counts, [L], L, N, hop, pad, torch.as_tensor(base)[None])
    assert torch.allclose(dw.v, x.grad[None] + torch.as_tensor(base)[None].double(), rtol=1e-9, atol=1e-9)
    assert torch.allclose(lm.v, mel.detach(), rtol=1e-12, atol=1e-12)
    return spec, lm, dw


def front_end_case(seed, scale_fb=1.0, amp=1.0):
    g = np.random.default_rng(seed)
    L = 3000
    wav = (amp * (g.random(L) - 0.5)).astype(f32)
    if amp == 1.0:
        wav[1200:2600] = 0                                                     # silent frames: |X| = sqrt(eps) exactly at the model's floor
    fb = (slaney_filterbank(GEO["sr"], GEO["N"], GEO["n_mels"]) * f32(scale_fb)).astype(f32)
    T = S.frames_of_row(L, (GEO["N"] - GEO["hop"]) // 2, GEO["N"], GEO["hop"])
    dmel = g.standard_normal((T, GEO["n_mels"])).astype(f32)
    base = g.standard_normal(L).astype(f32)
    return wav, fb, dmel, base


def test_front_end_and_adjoint_within_model(host):
    wav, fb, dmel, base = front_end_case(1)
    spec, lm, dw = pipeline(host, wav, fb, dmel, base)
    rs, rl, rd = reference(wav, fb, dmel, base)
    ws = within_model(torch.as_tensor(spec)[None], rs, "spec")
    wl = within_model(torch.as_tensor(lm)[None], rl, "log-mel")
    wd = within_model(torch.as_tensor(dw)[None], rd, "dwav")
    print(f"front end: worst err / model spec {ws * R.SAFETY:.3f}, log-mel {wl * R.SAFETY:.3f}, dwav {wd * R.SAFETY:.3f}")


@pytest.mark.parametrize("fault", ["frame start", "eps", "fb shift", "hermitian", "ola frame"])
def test_front_end_fault_outside_gate(host, fault):
    wav, fb, dmel, base = front_end_case(2)
    spec, lm, dw = pipeline(host, wav, fb, dmel, base, fault=fault)
    rs, rl, rd = reference(wav, fb, dmel, base)
    got, ref = {"frame start": (spec, rs), "eps": (spec, rs), "fb shift": (lm, rl)}.get(fault, (dw, rd))
    outside(torch.as_tensor(got)[None], ref, fault)


def test_clip_mask_fault_outside_gate(host):
    """a quiet row under a filterbank scaled by 0.1: every mel sits on the clip (lm == logf(clip)), so the gradient is 0;
    `>=` for `>` in the clip test passes dmel e^{-lm} instead"""
    wav, fb, dmel, base = front_end_case(3, scale_fb=0.1, amp=1e-6)
    rs, rl, rd = reference(wav, fb, dmel, base)
    assert bool((rl.v == math.log(S.CLIP)).all())
    _, _, ok = pipeline(host, wav, fb, dmel, base)
    within_model(torch.as_tensor(ok)[None], rd, "dwav on the clip")
    _, _, dw = pipeline(host, wav, fb, dmel, base, fault="clip >=")
    outside(torch.as_tensor(dw)[None], rd, "`>=` for `>` in the clip mask")


@pytest.mark.parametrize("fault", ["twiddle", "window j+1", "reflect about L"])
def test_transform_fault_outside_gate(host, fault):
    N, win, L = 2048, 2048, 5000
    wav = row(11, L)
    s0s = [-N // 2 + 3, 1500, L - N + 700]
    Xr, e = ref_X(wav, N, win, s0s)
    if fault == "twiddle":
        host[0].stft_set_fault(1, 0)
    elif fault == "window j+1":
        host[0].stft_set_fault(-1, 1)
    try:
        if fault == "reflect about L":                                      # i -> 2 L - i past the end; sample L reads 0
            X = []
            for s in s0s:
                i = np.abs(s + np.arange(N))
                fr = np.where(i >= L, np.where(2 * L - i < L, wav[np.minimum(2 * L - i, L - 1)], 0), wav[np.minimum(i, L - 1)])
                fr = np.ascontiguousarray(fr.astype(f32))
                X.append(frame_fwd(host, fr, N, 0, N, win))
            X = np.stack(X)
        else:
            X = np.stack([frame_fwd(host, wav, L, s, N, win) for s in s0s])
    finally:
        host[0].stft_set_fault(-1, 0)
    outside(cplx_t(X), as_E(Xr, e), fault)


# ---- inverse STFT -------------------------------------------------------------------------------------------------------------
def istft_f32(host, X, N, hop, mask=None, env_skip=None):
    """evk_istft on one row: G = X (* mask) * (1 or 2) / N, the adjoint transform, window, y / env in frame order (fp32)"""
    T, NB = X.shape
    inv = f32(1.0) / f32(N)
    sc = np.full(NB, f32(2) * inv, f32)
    sc[0] = sc[-1] = inv
    xr, xi = X.real.astype(f32), X.imag.astype(f32)
    if mask is not None:
        xr, xi = cmul(xr, xi, mask.real.astype(f32), mask.imag.astype(f32))
    G = (xr * sc).astype(f32) + 1j * (xi * sc).astype(f32)
    h = hann_f32(N, N)
    fr = np.stack([(frame_adj(host, G[t], N) * h).astype(f32) for t in range(T)])
    Lout = hop * (T - 1)
    q = np.arange(Lout) + N // 2
    y, env = np.zeros(Lout, f32), np.zeros(Lout, f32)
    for f in range(T):
        j = q - f * hop
        ok = (j >= 0) & (j < N)
        y[ok] = (y[ok] + fr[f, j[ok]]).astype(f32)
        if f != env_skip:
            env[ok] = (env[ok] + (h[j[ok]] * h[j[ok]]).astype(f32)).astype(f32)
    return (y / env).astype(f32)


ISTFT_SIZES = [(2048, 441), (256, 64), (320, 80), (640, 160), (960, 240)]


@pytest.mark.parametrize("N,hop", ISTFT_SIZES, ids=[f"N{n}-hop{h}" for n, h in ISTFT_SIZES])
def test_istft_within_model(host, N, hop):
    g = np.random.default_rng(N)
    T = 9
    NB = N // 2 + 1
    X = (g.standard_normal((T, NB)) + 1j * g.standard_normal((T, NB))).astype(np.complex64).astype(np.complex128)
    M = (g.standard_normal((T, NB)) + 1j * g.standard_normal((T, NB))).astype(np.complex64).astype(np.complex128)
    for mask in (None, M):
        got = istft_f32(host, X, N, hop, mask)
        ref, manual = S.istft(torch.as_tensor(X)[None], N, hop, None if mask is None else torch.as_tensor(mask)[None])
        assert torch.allclose(ref.v, manual, rtol=1e-9, atol=1e-12)
        w = within_model(torch.as_tensor(got)[None], ref, f"istft N={N} hop={hop} mask={mask is not None}")
        print(f"istft N={N} hop={hop} mask={mask is not None}: worst err / model {w * R.SAFETY:.3f}")


def test_istft_envelope_fault_outside_gate(host):
    N, hop, T = 2048, 441, 9
    g = np.random.default_rng(5)
    X = (g.standard_normal((T, N // 2 + 1)) + 1j * g.standard_normal((T, N // 2 + 1))).astype(np.complex64).astype(np.complex128)
    got = istft_f32(host, X, N, hop, env_skip=4)
    ref, _ = S.istft(torch.as_tensor(X)[None], N, hop)
    outside(torch.as_tensor(got)[None], ref, "envelope missing one frame")


def test_cplx_l1_emulation_within_model():
    g = torch.Generator().manual_seed(0)
    n = 132 * 8 * 256 + 777
    a, b = torch.randn(n, 2, generator=g), torch.randn(n, 2, generator=g)
    b[::97] = a[::97]
    d = (a - b).float()
    m = torch.sqrt((d * d).sum(-1).float()).float()
    sc = R.f32(1.0 / n)
    part = R.grid_partials(m, 132 * 8)
    loss = R.ordered_sum((part * sc).float()[:, None], torch.tensor([0.25]))
    grad = torch.where(m[:, None] > 0, d * (sc / m.clamp_min(1e-30)).float()[:, None], torch.zeros_like(d)).float()
    rl, rg = S.cplx_l1(a, b, float(sc), 0.25)
    within_model(loss, rl, "cplx_l1 loss")
    within_model(grad, rg, "cplx_l1 grad")
    assert bool((grad[::97] == 0).all())
