"""Float64 references and per-element error bounds for the fp32 spectral kernels (csrc/mel.cu: the warp-per-frame log-mel front
end and spec_to_mel; csrc/stft.cu: the general STFT, its adjoint, the inverse STFT and the complex L1 loss), for
tests/test_gpu_spectral_elementwise.py; tests/test_cpu_spectral_ref.py rehearses them against fp32 emulations of the kernels.

References: reflect pad (at each row's own end), frames, the exact periodic Hann window, torch.fft.rfft, sqrt(re^2 + im^2 + eps),
the fp32 Slaney filterbank promoted to float64, log(clamp(., clip)), the backward by float64 autograd of the same expression,
torch.istft and the complex L1 loss, all in float64.  eps and clip are the fp32 constants the kernels use.

Error model (the conventions of tests/cudacore_ref.py: U32 = 2^-24 per correctly rounded fp32 operation, the CUDA ulp tables
for logf / expf, gate = SAFETY x model, nothing fitted to a GPU measurement).
- FFT.  Every intermediate of a Stockham pass (and of the warp kernel's radix-2 stages) is a partial DFT of the even/odd-packed
  frame d[m] = (a[2m], a[2m+1]), a[n] = x[n] w[n], over a subset of the m, times unit-modulus twiddles, so its modulus is at most
  the sum of |d[m]| over that subset, and every later operation carries its error to an output with a coefficient of modulus 1.
  The subsets of one pass partition the frame, so a pass adds at most c_pass * u * sum|d| <= c_pass * u * sum|a| to every
  output.  A complex multiply by an fp32 table twiddle costs CMUL = 2 sqrt(2) + 1: 2 sqrt(2) u |v| for the multiply in either
  form (plain: two products and a sum per component; FMA-contracted: one product and an fma), u |v| for the table entry.
  c_pass: radix 4: CMUL (the three twiddles) + 2 (two addition levels), 2 in the first pass (no twiddle); radix 2: CMUL + 1,
  1 in the first pass; radix 3 / 5: 2 CMUL (twiddle and root) + R - 1 additions, CMUL + R - 1 in the first pass.  The warp
  kernel's 32 x 32 decomposition: 5 radix-2 DIF stages (CMUL + 1 each: a difference, then the fmaf twiddle by an fp32
  constant), CMUL for the inter-stage twiddle, 5 more stages.  The untangle mixes Z[k] and conj(Z[NH-k]) with coefficients
  (1 -+ i w) / 2 whose squared moduli sum to 1, so it carries the FFT error times sqrt(2) and adds CMUL + 4 of its own (two
  halved sums, the twiddle, the final sum of modulus <= 2 sum|d|).  The window adds 2 u |a[n]| (the table and the product).
  Hence |dX_k| <= (2 + sqrt(2) c_fft + CMUL + 4) u sum|a|, one bound per frame.
- |X| = sqrtf(re^2 + im^2 + eps): 1-Lipschitz in X, plus 3 roundings of the radicand (half of them after the root) and the
  root: 2.5 u |X|.  eps >= 1e-6 keeps |X| >= 1e-3, which bounds the X / |X| conditioning of the adjoint.
- mel = logf(fmaxf(sum_e val_e |X|_idx_e, clip)): the fmaf chain runs in CSR order (bins ascending), so term e is rounded into
  every partial sum from e to the end of its row: u * sum_e val_e |X|_idx_e (p1 - e).  fmaxf is 1-Lipschitz; logf: 1 ulp.
- adjoint, log-mel path: g_m = dmel e^{-lm} (expf: 2 ulp, and the forward's error of lm); a mel whose float64 sum lies within
  SAFETY x its bound of the clip may fall on either side of the kernel's `lm > log(clip)` test, so its whole g_m joins the
  error; dmag_k = sum_m val g_m in mel order (count + 1 roundings); G_k = dmag_k X_k / |X_k| with the kernel's own X:
  |dG| <= (|d dmag| + 4.5 u |dmag|) |X| / |X|_eps + 2 |dmag| |dX| / |X|_eps.  The inverse transform S[n] = sum_k Re(G_k e^{+2 pi i k n / N}) has
  unit-modulus coefficients: |dS| <= sum_k |dG_k| + (CMUL + 4 + 2 c_fft) u sum_k |G_k| (the packing, then the forward FFT of
  the packed sequence, whose moduli sum to at most 2 sum|G|).  The window adds 2 u w |S|.  The overlap-add gathers the
  terms of a sample in a fixed order: terms * u * sum |terms|, then u (|base| + sum |terms|) for the += onto the dwav base
  (exact when every term is 0, as on a silent row).
- iSTFT: G = X * mask * (1 or 2) / N (2 sqrt(2) + 2 u |G|), the same inverse transform and window, then y / env with
  env = sum w^2 (3 u w^2 a term) over the same frames.
Frames past a row's own count, the samples at n >= Lrow and pitch padding are exact (bound 0).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from tests.cudacore_ref import E, F64, NUM_SMS, SAFETY, TINY, U32, ULP, ULPS, grid_reduce_chain

CMUL = 2.0 * math.sqrt(2.0) + 1.0
EPS = float(np.float32(1e-6))          # the kernels' fp32 magnitude eps and log clip
CLIP = float(np.float32(1e-5))
TAB, TAB_MR = 4096, 4096 * 15


# ---- geometry ---------------------------------------------------------------------------------------------------------------
def frames_of_row(Lrow, pad, N, hop):
    """frames of a row of Lrow valid samples: none when it is too short to reflect once (Lrow <= pad)"""
    span = Lrow + 2 * pad - N
    return 0 if (span < 0 or Lrow <= pad) else span // hop + 1


def stockham_passes(NH):
    """[(R, Ns)] of stft_core.cuh's stft_radix: radix 4 while it divides what is left, then 2, 3, 5"""
    out, Ns = [], 1
    while Ns < NH:
        rem = NH // Ns
        R = 4 if rem % 4 == 0 else 2 if rem % 2 == 0 else 3 if rem % 3 == 0 else 5
        out.append((R, Ns))
        Ns *= R
    return out


def c_pass(R, first):
    if R == 4:
        return 2.0 if first else CMUL + 2.0
    if R == 2:
        return 1.0 if first else CMUL + 1.0
    return (CMUL if first else 2.0 * CMUL) + (R - 1)


def c_fft(N, warp=False):
    """the FFT of the N/2-point packed sequence: sum of the passes' counts"""
    if warp:
        assert N == 2048
        return 10 * (CMUL + 1.0) + CMUL
    return sum(c_pass(R, Ns == 1) for R, Ns in stockham_passes(N // 2))


def c_forward(N, warp=False):
    """|dX_k| <= c_forward * u * sum|a|: window, FFT carried through the untangle, the untangle's own roundings"""
    return 2.0 + math.sqrt(2.0) * c_fft(N, warp) + CMUL + 4.0


def c_inverse(N):
    """rounding of the adjoint packing and its forward FFT, per unit of sum_k |G_k|"""
    return CMUL + 4.0 + 2.0 * c_fft(N)


# ---- forward --------------------------------------------------------------------------------------------------------------
def hann(win):
    """periodic Hann(win) in float64 (torch.hann_window(win), exact)"""
    return 0.5 - 0.5 * torch.cos(2.0 * math.pi * torch.arange(win, dtype=F64) / win)


def window(N, win):
    """Hann(win) centred in the N-point frame, zero outside (torch.stft's padding of a short window)"""
    w = torch.zeros(N, dtype=F64)
    off = (N - win) // 2
    w[off:off + win] = hann(win)
    return w


def row_frames(x, Lrow, N, hop, pad, T):
    """[T, N] windowless frames of one row x [>= Lrow] reflect-padded at its own end; rows past its own count are zero.
    Differentiable wrt x."""
    Tr = frames_of_row(Lrow, pad, N, hop)
    assert Tr <= T
    out = [torch.zeros(T - Tr, N, dtype=F64)]
    if Tr:
        xr = x[:Lrow]
        xp = F.pad(xr[None, None], (pad, pad), mode="reflect")[0, 0] if pad else xr
        out.insert(0, xp.unfold(0, N, hop)[:Tr])
    return torch.cat(out, 0), Tr


def stft(wav, lens, N, hop, win, pad, T):
    """wav [B, L] float64 -> X [B, T, N/2+1] complex128, A [B, T] = sum_n |x_n w_n|, counts [B]"""
    B, L = wav.shape
    w = window(N, win)
    Xs, As, Ts = [], [], []
    for b in range(B):
        Lr = L if lens is None else min(int(lens[b]), L)
        fr, Tr = row_frames(wav[b], Lr, N, hop, pad, T)
        a = fr * w
        Xs.append(torch.fft.rfft(a))
        As.append(a.detach().abs().sum(-1))
        Ts.append(Tr)
    return torch.stack(Xs), torch.stack(As), Ts


def magnitude(X):
    return torch.sqrt(X.real ** 2 + X.imag ** 2 + EPS)


def e_forward(A, N, warp=False):
    """[B, T, 1] bound of every bin of X"""
    return (c_forward(N, warp) * U32 * A)[..., None]


def spec_E(X, A, N, warp=False):
    m = magnitude(X).detach()
    return E(m, e_forward(A, N, warp) + 2.5 * U32 * m + TINY)


def csr_weights(fb):
    """[n_mels, n_bins]: for a non-zero of row m, the number of partial sums of the CSR fmaf chain it is rounded into"""
    nz = (fb != 0).to(F64)
    return torch.flip(torch.cumsum(torch.flip(nz, [1]), 1), [1]) * nz


def mel_sum(spec, fb):
    """the filterbank sum of an E spectrum (..., n_bins) in CSR order: E (..., n_mels)"""
    fb = fb.to(F64)
    v = spec.v @ fb.T
    return E(v, spec.e @ fb.T + U32 * (spec.v @ (fb * csr_weights(fb)).T) + TINY)


def log_clip(s):
    """logf(fmaxf(s, clip)): E"""
    c = s.v.clamp_min(CLIP)
    v = torch.log(c)
    return E(v, s.e / c + ULPS["log"] * (ULP * v.abs() + TINY))


def logmel_value(spec_v, fb):
    return torch.log(torch.clamp(spec_v @ fb.to(F64).T, min=CLIP))


# ---- adjoint ---------------------------------------------------------------------------------------------------------------
def mel_adjoint_G(X, A, N, fb, dmel, warp=False):
    """G [B, T, NB] complex (the float64 gradient wrt X of sum dmel * logmel) and its bound e_G, with the forward errors of the
    kernel's own saved cplx (X) and mel, and the clip test taken either way where it is ambiguous"""
    fb = fb.to(F64)
    eX = e_forward(A, N, warp)
    spec = spec_E(X, A, N, warp)
    s = mel_sum(spec, fb)
    lm = log_clip(s)
    live = s.v > CLIP
    amb = (s.v - CLIP).abs() <= SAFETY * s.e
    gm = torch.where(live, dmel * torch.exp(-lm.v), torch.zeros_like(dmel))
    e_gm = gm.abs() * (lm.e + ULPS["exp"] * ULP + U32) + torch.where(amb, (dmel * torch.exp(-lm.v)).abs(), torch.zeros_like(dmel))
    dmag = gm @ fb
    cnt = (fb != 0).sum(0).to(F64)
    e_dmag = e_gm @ fb + (cnt + 1) * U32 * (gm.abs() @ fb)
    m = magnitude(X)
    G = dmag * X / m
    r = X.abs() / m                                                           # |G| / |dmag| <= 1: exactly 0 on a silent frame
    e_G = (e_dmag + 4.5 * U32 * dmag.abs()) * r + 2.0 * dmag.abs() * eX / m
    return G, e_G


def inverse_frames(G, e_G, N, win):
    """S[n] w[n] of every frame (the windowed adjoint the kernel overlap-adds) and its bound: [..., N] each"""
    w = window(N, win)
    # S[n] = sum_k Re(G_k e^{+2 pi i k n / N}) over k = 0 .. N/2 = irfft(G') * N with G'_k = G_k / 2 inside, real G_0, G_NH
    Gp = G.clone()
    Gp[..., 1:-1] = Gp[..., 1:-1] / 2
    S = torch.fft.irfft(Gp, n=N) * N
    Mg = G.abs().sum(-1, keepdim=True)
    eS = e_G.sum(-1, keepdim=True) + c_inverse(N) * U32 * Mg
    return S * w, w * eS + 2.0 * U32 * w * Mg


def fold_index(Lrow, N, hop, pad, Tr):
    """[Tr, N] sample index each frame position reads (reflect at the row's own end)"""
    s = torch.arange(Tr)[:, None] * hop - pad + torch.arange(N)[None, :]
    s = s.abs()
    s = torch.where(s >= Lrow, 2 * (Lrow - 1) - s, s)
    assert bool((s >= 0).all()) and bool((s < Lrow).all())
    return s


def ola(frames, e_frames, counts, lens_eff, L, N, hop, pad, base):
    """dwav [B, L] = base + the overlap-add of each row's own frames through the reflect index, and its bound"""
    B = frames.shape[0]
    v = base.to(F64).clone()
    mag = torch.zeros(B, L, dtype=F64)
    err = torch.zeros(B, L, dtype=F64)
    nterm = torch.zeros(B, L, dtype=F64)
    for b in range(B):
        Tr, Lr = counts[b], lens_eff[b]
        if Tr == 0:
            continue
        idx = fold_index(Lr, N, hop, pad, Tr).reshape(-1)
        v[b].index_add_(0, idx, frames[b, :Tr].reshape(-1))
        mag[b].index_add_(0, idx, frames[b, :Tr].abs().reshape(-1))
        err[b].index_add_(0, idx, e_frames[b, :Tr].expand(Tr, N).reshape(-1))
        nterm[b].index_add_(0, idx, torch.ones(Tr * N, dtype=F64))
    e = err + nterm * U32 * mag + U32 * (mag + base.to(F64).abs()) * (mag > 0)     # base + 0 is exact
    return E(v, e)


# ---- inverse STFT ----------------------------------------------------------------------------------------------------------
def istft(X, N, hop, mask_c=None):
    """X [R, T, NB] complex128 (times mask_c when given) -> E [R, hop (T - 1)]: torch.istft(center=True, Hann(N)) and its bound"""
    Xm = X if mask_c is None else X * mask_c
    R_, T, NB = Xm.shape
    w = hann(N)
    out = torch.istft(Xm.transpose(1, 2), N, hop, N, window=w, center=True, normalized=False, onesided=True)
    sc = torch.full((NB,), 2.0 / N, dtype=F64)
    sc[0] = sc[-1] = 1.0 / N
    G = Xm * sc
    e_G = G.abs() * ((2.0 * math.sqrt(2.0) if mask_c is not None else 0.0) + 2.0) * U32
    S = torch.fft.irfft(Xm, n=N)                                              # [R, T, N]
    Mg = G.abs().sum(-1, keepdim=True)
    eS = e_G.sum(-1, keepdim=True) + c_inverse(N) * U32 * Mg
    fr, efr = S * w, w * eS + 2.0 * U32 * w * Mg
    Lout = hop * (T - 1)
    q = torch.arange(Lout) + N // 2
    y = torch.zeros(R_, Lout, dtype=F64)
    ey = torch.zeros(R_, Lout, dtype=F64)
    my = torch.zeros(R_, Lout, dtype=F64)
    env = torch.zeros(Lout, dtype=F64)
    cnt = torch.zeros(Lout, dtype=F64)
    for f in range(T):
        j = q - f * hop
        ok = (j >= 0) & (j < N)
        jj = j[ok]
        y[:, ok] += fr[:, f, jj]
        ey[:, ok] += efr[:, f, jj]
        my[:, ok] += fr[:, f, jj].abs()
        env[ok] += w[jj] ** 2
        cnt[ok] += 1
    e_y = ey + cnt * U32 * my
    e_env = (3.0 + cnt) * U32 * env
    o = y / env
    return E(out, e_y / env + o.abs() * e_env / env + U32 * o.abs() + TINY), y / env


# ---- complex L1 -------------------------------------------------------------------------------------------------------------
def cplx_l1(a, b, scale, base):
    """a, b [n, 2] fp32: loss base + scale sum |a - b| (block_sum, then ordered_sum over the <= 132 * 8 blocks) and
    grad scale (a - b) / |a - b| (exactly 0 where a == b)"""
    d = a.double() - b.double()
    m = torch.sqrt((d * d).sum(-1))
    n = a.shape[0]
    chain = grid_reduce_chain(n, NUM_SMS * 8)
    sc = float(np.float32(scale))
    tot = sc * m.sum()
    loss = E(base + tot, sc * 3.5 * U32 * m.sum() + chain * U32 * (tot.abs() + abs(base)) + TINY)
    g = torch.where(m[:, None] > 0, sc * d / m.clamp_min(1e-300)[:, None], torch.zeros_like(d))
    grad = E(g, 6.5 * U32 * g.abs() + TINY * (m[:, None] > 0))
    return loss, grad
