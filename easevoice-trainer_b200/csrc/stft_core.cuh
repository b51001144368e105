// Core of the general STFT kernels: one thread block per frame, Stockham passes of radix 4, 2, 3 and 5 over the even/odd-packed
// frame in shared memory.  Everything here is `EVK_HD` so that the host harnesses under tools/exp can run the very same index
// arithmetic on the host (threads emulated by a loop, barriers by phase boundaries) against numpy.
//
// Conventions: N = n_fft, NH = N / 2.  Tables are indexed in units of 2 pi / tab:
//   tw[i]   = (cos(2 pi i / tab), -sin(2 pi i / tab)),  i < tab         (forward twiddles)
//   hann[i] = 0.5 - 0.5 cos(2 pi i / tab),              i < tab         (periodic Hann of length tab; a window of length `win`
//             dividing tab is hann[j * (tab / win)], exactly torch.hann_window(win)[j] up to fp32 rounding)
// Two tables exist: STFT_TAB = 8192 serves the power-of-two sizes (n_fft 256 .. 8192, radix 4 plus one radix-2 pass), and
// STFT_TAB_MR = 4096 * 15 every even N dividing it, i.e. N = 2^a 3^b 5^c with a <= 12, b, c <= 1 (the UVR5 band sizes
// 320, 640, 960 among them).  The functions without a `tab` argument are the power-of-two ones on STFT_TAB.  Entry j * 2 of the
// 8192-entry tables is bit for bit entry j of a 4096-entry one (2 pi (2j) / 8192 and 2 pi j / 4096 are the same double), and
// every index scales with tab, so the sizes up to 4096 compute exactly what they did on 4096-entry tables.
#pragma once

#ifndef EVK_HD
#ifdef __CUDACC__
#define EVK_HD __host__ __device__ __forceinline__
#else
#define EVK_HD inline
#endif
#endif

namespace evk {

constexpr int STFT_TAB = 8192;
constexpr int STFT_TAB_MR = 4096 * 15;

EVK_HD float2 stft_cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

EVK_HD int stft_reflect(int i, int L) {
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  if (i < 0) i = 0;                       // only for rows no longer than the padding: stft.cu gives those no frames, so
                                          // there it is unreachable; vr_wave.cu's reflect mode reaches it for bands of
                                          // <= n_fft / 2 samples
  return i;
}

// window value at position n of the n_fft-long frame: periodic Hann(win) centred in the frame (torch.stft pads the
// window on both sides to n_fft), zero outside
EVK_HD float stft_window_t(const float* hann, int n, int N, int win, int tab) {
  const int off = (N - win) >> 1, j = n - off;
  return (j >= 0 && j < win) ? hann[j * (tab / win)] : 0.f;
}
EVK_HD float stft_window(const float* hann, int n, int N, int win) { return stft_window_t(hann, n, N, win, STFT_TAB); }

// ---- phase: load + window + even/odd pack:  d[m] = (x[2m] w[2m], x[2m+1] w[2m+1]),  m = tid, tid+nt, ... < NH ---------
// zero_pad: samples outside [0, Lrow) read as 0 (librosa >= 0.9's pad_mode="constant") instead of reflecting
EVK_HD float stft_sample(const float* wav, int i, int Lrow, bool zero_pad) {
  if (zero_pad) return (i >= 0 && i < Lrow) ? wav[i] : 0.f;
  return wav[stft_reflect(i, Lrow)];
}
EVK_HD void stft_load_phase_t(int tid, int nt, const float* wav, int Lrow, int s0, int N, int win, const float* hann, int tab, bool zero_pad,
                              float2* d) {
  const int NH = N >> 1;
  for (int m = tid; m < NH; m += nt) {
    const int n0 = 2 * m, n1 = n0 + 1;
    const float w0 = stft_window_t(hann, n0, N, win, tab), w1 = stft_window_t(hann, n1, N, win, tab);
    const float a = (w0 != 0.f) ? stft_sample(wav, s0 + n0, Lrow, zero_pad) * w0 : 0.f;
    const float b = (w1 != 0.f) ? stft_sample(wav, s0 + n1, Lrow, zero_pad) * w1 : 0.f;
    d[m] = make_float2(a, b);
  }
}
EVK_HD void stft_load_phase(int tid, int nt, const float* wav, int Lrow, int s0, int N, int win, const float* hann, float2* d) {
  stft_load_phase_t(tid, nt, wav, Lrow, s0, N, win, hann, STFT_TAB, false, d);
}

// ---- radix of the pass after the first Ns points are done: 4 while it divides what is left, then 2, 3, 5 ---------------------
// (for a power of two: radix 4 while Ns * 4 <= NH, then one radix-2 pass when log2(NH) is odd)
EVK_HD int stft_radix(int NH, int Ns) {
  const int rem = NH / Ns;
  return (rem % 4 == 0) ? 4 : (rem % 2 == 0) ? 2 : (rem % 3 == 0) ? 3 : 5;
}

// ---- one Stockham pass of radix R of the NH-point complex FFT (forward, e^{-i...}) with twiddles of table size tab --------
// stft_radix takes the factors 2 first, so Ns is a power of two in every radix-4 and radix-2 pass.
// Returns the new Ns = Ns * R.  All threads must call it with the same arguments; a barrier is needed after each pass.
EVK_HD int stft_pass_r(int tid, int nt, int NH, int Ns, int R, const float2* src, float2* dst, const float2* tw, int tab) {
  if (R == 4) {
    const int Q = NH >> 2, tstep = tab / (4 * Ns);
    for (int j = tid; j < Q; j += nt) {
      const int k = j & (Ns - 1);
      float2 v0 = src[j], v1 = src[j + Q], v2 = src[j + 2 * Q], v3 = src[j + 3 * Q];
      if (Ns > 1) {
        v1 = stft_cmul(v1, tw[k * tstep]);
        v2 = stft_cmul(v2, tw[2 * k * tstep]);
        v3 = stft_cmul(v3, tw[3 * k * tstep]);
      }
      const float2 a0 = make_float2(v0.x + v2.x, v0.y + v2.y), a1 = make_float2(v0.x - v2.x, v0.y - v2.y);
      const float2 a2 = make_float2(v1.x + v3.x, v1.y + v3.y);
      const float2 t = make_float2(v1.x - v3.x, v1.y - v3.y);
      const float2 a3 = make_float2(t.y, -t.x);        // (v1 - v3) * (-i)
      const int idx = (j / Ns) * Ns * 4 + k;
      dst[idx] = make_float2(a0.x + a2.x, a0.y + a2.y);
      dst[idx + Ns] = make_float2(a1.x + a3.x, a1.y + a3.y);
      dst[idx + 2 * Ns] = make_float2(a0.x - a2.x, a0.y - a2.y);
      dst[idx + 3 * Ns] = make_float2(a1.x - a3.x, a1.y - a3.y);
    }
    return Ns * 4;
  }
  if (R == 2) {
    const int H = NH >> 1, tstep = tab / (2 * Ns);
    for (int j = tid; j < H; j += nt) {
      const int k = j & (Ns - 1);
      const float2 v0 = src[j];
      float2 v1 = src[j + H];
      if (Ns > 1) v1 = stft_cmul(v1, tw[k * tstep]);
      const int idx = (j / Ns) * Ns * 2 + k;
      dst[idx] = make_float2(v0.x + v1.x, v0.y + v1.y);
      dst[idx + Ns] = make_float2(v0.x - v1.x, v0.y - v1.y);
    }
    return Ns * 2;
  }
  // odd radix (3 or 5): twiddle, then an R-point DFT whose roots e^{-2 pi i q / R} are table entries q * tab / R
  const int Q = NH / R, tstep = tab / (R * Ns), rstep = tab / R;
  for (int j = tid; j < Q; j += nt) {
    const int k = j % Ns;
    float2 v[5];
    for (int r = 0; r < R; ++r) {
      v[r] = src[j + r * Q];
      if (Ns > 1 && r > 0) v[r] = stft_cmul(v[r], tw[r * k * tstep]);
    }
    const int idx = (j / Ns) * Ns * R + k;
    for (int m = 0; m < R; ++m) {
      float2 acc = v[0];
      for (int r = 1; r < R; ++r) {
        const float2 p = stft_cmul(v[r], tw[((r * m) % R) * rstep]);
        acc = make_float2(acc.x + p.x, acc.y + p.y);
      }
      dst[idx + m * Ns] = acc;
    }
  }
  return Ns * R;
}

// the power-of-two pass on STFT_TAB (radix 4 when Ns * 4 <= NH, else radix 2)
EVK_HD int stft_pass(int tid, int nt, int NH, int Ns, const float2* src, float2* dst, const float2* tw) {
  return stft_pass_r(tid, nt, NH, Ns, (Ns * 4 <= NH) ? 4 : 2, src, dst, tw, STFT_TAB);
}

// ---- phase: real-FFT untangle  X[k] = (Z[k] + conj(Z[NH-k]))/2 - (i/2) e^{-2 pi i k/N} (Z[k] - conj(Z[NH-k])), k <= NH ----
EVK_HD void stft_untangle_phase_t(int tid, int nt, int N, const float2* z, const float2* tw, int tab, float2* X) {
  const int NH = N >> 1, step = tab / N;
  for (int k = tid; k <= NH; k += nt) {
    const float2 zk = z[k == NH ? 0 : k];
    float2 zc = z[k == 0 ? 0 : NH - k];
    zc.y = -zc.y;
    const float2 s = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
    const float2 dd = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
    const float2 w = (k < NH) ? tw[k * step] : make_float2(-1.f, 0.f);      // e^{-i pi} at k = NH (index TAB/2 also works; explicit for N = TAB)
    const float2 t = stft_cmul(w, dd);
    X[k] = make_float2(s.x + t.y, s.y - t.x);        // s - i t
  }
}
EVK_HD void stft_untangle_phase(int tid, int nt, int N, const float2* z, const float2* tw, float2* X) {
  stft_untangle_phase_t(tid, nt, N, z, tw, STFT_TAB, X);
}

// ---- adjoint: given G[k] = dL/dRe X[k] + i dL/dIm X[k] (k <= NH), build conj(Z'') so that ONE MORE forward FFT yields
//      S[n] = sum_k Re(G[k] e^{+2 pi i k n / N}) = dL/d(x[n] w[n]):   S[2m] = r[m].x, S[2m+1] = -r[m].y -------
EVK_HD void stft_adjoint_pack_phase_t(int tid, int nt, int N, const float2* G, const float2* tw, int tab, float2* d) {
  const int NH = N >> 1, step = tab / N;
  for (int k = tid; k < NH; k += nt) {
    // F[0] = Re G[0], F[NH] = Re G[NH], F[k] = G[k] / 2 otherwise (Hermitian completion of the one-sided gradient)
    float2 A = G[k], B = G[NH - k];
    if (k == 0) { A = make_float2(A.x, 0.f); B = make_float2(B.x, 0.f); }
    else { A = make_float2(0.5f * A.x, 0.5f * A.y); B = make_float2(0.5f * B.x, 0.5f * B.y); }
    const float2 Bc = make_float2(B.x, -B.y);
    const float2 s = make_float2(A.x + Bc.x, A.y + Bc.y), dd = make_float2(A.x - Bc.x, A.y - Bc.y);
    const float2 w = tw[k * step];                   // e^{-i phi}; e^{+i phi} = conj
    const float2 e = stft_cmul(make_float2(w.x, -w.y), dd);
    const float2 Z = make_float2(s.x - e.y, s.y + e.x);   // s + i e
    d[k] = make_float2(Z.x, -Z.y);                    // conj: inverse FFT = conj(forward FFT(conj(.)))
  }
}
EVK_HD void stft_adjoint_pack_phase(int tid, int nt, int N, const float2* G, const float2* tw, float2* d) {
  stft_adjoint_pack_phase_t(tid, nt, N, G, tw, STFT_TAB, d);
}

// ---- supported mixed-radix frame sizes: even N dividing STFT_TAB_MR, 16 <= N <= 7680 (shared memory of one block) -------
EVK_HD bool stft_mr_size_ok(int N) { return N >= 16 && N <= 7680 && N % 2 == 0 && STFT_TAB_MR % N == 0; }

}  // namespace evk
