// Core of the general STFT kernels (n_fft = 256 .. 4096, any hop, win <= n_fft, center or not): one thread block per frame,
// Stockham radix-4 (+ one radix-2 pass when log2(n_fft/2) is odd) over the even/odd-packed frame in shared memory.
// Everything here is `EVK_HD` so that tools/exp/stft_host_test.cpp can run the very same index arithmetic on the host
// (threads emulated by a loop, barriers by phase boundaries) against numpy -- there is no GPU in the authoring container.
//
// Conventions: N = n_fft, NH = N / 2.  Tables are indexed in units of 2 pi / TAB (TAB = 4096):
//   tw[i]   = (cos(2 pi i / TAB), -sin(2 pi i / TAB)),  i < TAB         (forward twiddles)
//   hann[i] = 0.5 - 0.5 cos(2 pi i / TAB),              i < TAB         (periodic Hann of length TAB; a power-of-two
//             window of length `win` is hann[j * (TAB / win)], exactly torch.hann_window(win)[j] up to fp32 rounding)
#pragma once

#ifndef EVK_HD
#ifdef __CUDACC__
#define EVK_HD __host__ __device__ __forceinline__
#else
#define EVK_HD inline
#endif
#endif

namespace evk {

constexpr int STFT_TAB = 4096;

EVK_HD float2 stft_cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

EVK_HD int stft_reflect(int i, int L) {
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  if (i < 0) i = 0;                       // only for rows shorter than the padding (never the case for real inputs)
  return i;
}

// window value at position n of the n_fft-long frame: periodic Hann(win) centred in the frame (torch.stft pads the
// window on both sides to n_fft), zero outside
EVK_HD float stft_window(const float* hann, int n, int N, int win) {
  const int off = (N - win) >> 1, j = n - off;
  return (j >= 0 && j < win) ? hann[j * (STFT_TAB / win)] : 0.f;
}

// ---- phase: load + window + even/odd pack:  d[m] = (x[2m] w[2m], x[2m+1] w[2m+1]),  m = tid, tid+nt, ... < NH ---------
EVK_HD void stft_load_phase(int tid, int nt, const float* wav, int Lrow, int s0, int N, int win, const float* hann, float2* d) {
  const int NH = N >> 1;
  for (int m = tid; m < NH; m += nt) {
    const int n0 = 2 * m, n1 = n0 + 1;
    const float w0 = stft_window(hann, n0, N, win), w1 = stft_window(hann, n1, N, win);
    const float a = (w0 != 0.f) ? wav[stft_reflect(s0 + n0, Lrow)] * w0 : 0.f;
    const float b = (w1 != 0.f) ? wav[stft_reflect(s0 + n1, Lrow)] * w1 : 0.f;
    d[m] = make_float2(a, b);
  }
}

// ---- one Stockham pass of the NH-point complex FFT (forward, e^{-i...}).  radix 4 when Ns * 4 <= NH else radix 2. ------
// Returns the new Ns.  All threads must call it with the same arguments; a barrier is needed after each pass.
EVK_HD int stft_pass(int tid, int nt, int NH, int Ns, const float2* src, float2* dst, const float2* tw) {
  if (Ns * 4 <= NH) {
    const int Q = NH >> 2, tstep = STFT_TAB / (4 * Ns);
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
  const int H = NH >> 1, tstep = STFT_TAB / (2 * Ns);
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

// ---- phase: real-FFT untangle  X[k] = (Z[k] + conj(Z[NH-k]))/2 - (i/2) e^{-2 pi i k/N} (Z[k] - conj(Z[NH-k])), k <= NH ----
EVK_HD void stft_untangle_phase(int tid, int nt, int N, const float2* z, const float2* tw, float2* X) {
  const int NH = N >> 1, step = STFT_TAB / N;
  for (int k = tid; k <= NH; k += nt) {
    const float2 zk = z[k & (NH - 1)];
    float2 zc = z[(NH - k) & (NH - 1)];
    zc.y = -zc.y;
    const float2 s = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
    const float2 dd = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
    const float2 w = (k < NH) ? tw[k * step] : make_float2(-1.f, 0.f);      // e^{-i pi} at k = NH (index TAB/2 also works; explicit for N = TAB)
    const float2 t = stft_cmul(w, dd);
    X[k] = make_float2(s.x + t.y, s.y - t.x);        // s - i t
  }
}

// ---- adjoint: given G[k] = dL/dRe X[k] + i dL/dIm X[k] (k <= NH), build conj(Z'') so that ONE MORE forward FFT yields
//      S[n] = sum_k Re(G[k] e^{+2 pi i k n / N}) = dL/d(x[n] w[n]):   S[2m] = r[m].x, S[2m+1] = -r[m].y -------
EVK_HD void stft_adjoint_pack_phase(int tid, int nt, int N, const float2* G, const float2* tw, float2* d) {
  const int NH = N >> 1, step = STFT_TAB / N;
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

}  // namespace evk
