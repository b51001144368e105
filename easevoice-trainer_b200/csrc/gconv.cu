// Generalised 1-D convolution / GEMM on tensor cores (TF32 operands, FP32 accumulate), channels-last.
//
//   Y[z][(o0 + j*os)*P + w][n] = epi( sum_q sum_c X[z][(j*is + off[q])*P + w][c] * W[z][q][n][c] )
//
// Forward kernel ("F"): output positions on the MMA M axis, output channels on N, input channels on K.
// The input rows a tile needs for ALL taps are staged once per channel chunk as a shared-memory slab
// (tap q reads the slab shifted by off[q]*P rows), so the implicit im2col never touches L2 twice.
// Weight-gradient kernel ("W"): positions on K, (n, c) on M/N, per-CTA partials added in a fixed order for the split-K merge.
//
// Replaces the cuDNN / cuBLAS kernels behind the reference's Conv1d / Conv2d(k,1) / ConvTranspose1d /
// Linear / matmul call sites (see include/evk.h for file:line).
#include "evk_common.cuh"

namespace evk {

constexpr int BM = 128;        // output positions per CTA (F kernel)
constexpr int NT = 256;        // threads per CTA

struct GP {
  const float* x; float* w; float* y; const float* res; const float* bias;
  const int* in_len; const int* out_len;
  long long x_sb, x_sh, w_sb, w_sh, w_sq, y_sb, y_sh, r_sb, r_sh;
  int ldx, ldw, ldy, ldr, b_sh;
  int Z, H, C, N, Q, Tin, J, P, is, os, o0, Tout, act;
  float slope;
  int off_min, off_max;
  int KS, TG, NG, slab_rows;   // F: k-steps/tap/chunk, taps per group, groups, slab rows
  int rch;                     // W: positions per CTA
  float* part;                 // W: per-(z, position chunk, K warp) partials [z - zoff][S1][Q][N][C], summed by gconv_w_sum
  int zoff;                    // W: first batch x group item of this launch (blockIdx.z counts from it)
  int off[EVK_MAX_TAPS];
};

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == EVK_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == EVK_ACT_RELU) return fmaxf(v, 0.f);
  if (act == EVK_ACT_TANH) return tanhf(v);
  if (act == EVK_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

// ============================================================================================
// F kernel
// ============================================================================================
// PRECISE: 3xTF32 error-compensated products (a = hi + lo), ~fp32 accuracy at 3x the tensor work; used by the
// parity tests to separate indexing errors from TF32 rounding, and selectable at run time (evk_set_precise).
template <int WARPS_M, int WARPS_N, int MF, int NF, bool PRECISE>
__global__ void __launch_bounds__(NT) gconv_f_kernel(const __grid_constant__ GP p) {
  static_assert(WARPS_M * WARPS_N * 32 == NT, "8 warps");
  static_assert(WARPS_M * MF * 16 == BM, "BM");
  constexpr int BN = WARPS_N * NF * 8;
  extern __shared__ __align__(16) float smem[];
  const int CK = p.KS * 8, LD = CK + 4, PCS = CK / 4;
  float* slab0 = smem;                                   // [2][slab_rows][LD]
  const int slab_sz = p.slab_rows * LD;
  float* wt0 = smem + 2 * slab_sz;                       // [2][TG][BN][LD]
  const int wt_sz = p.TG * BN * LD;
  __shared__ int s_base[BM];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gid = lane >> 2, t4 = lane & 3;
  const int wm = warp / WARPS_N, wn = warp % WARPS_N;
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const float* X = p.x + b * p.x_sb + h * p.x_sh;
  const float* Wg = p.w + b * p.w_sb + h * p.w_sh;
  const int p0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int npos = p.J * p.P;
  const int j_first = p0 / p.P;
  const int lo = (j_first * p.is + p.off_min) * p.P;
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  const int lim_rows = lim * p.P;

  for (int m = tid; m < BM; m += NT) {
    int pos = p0 + m, v = 0;
    if (pos < npos) {
      int j = pos / p.P, w = pos - j * p.P;
      v = (j * p.is + p.off_min) * p.P + w - lo;
    }
    s_base[m] = v;
  }

  const int nchunks = (p.C + CK - 1) / CK;
  const int U = nchunks * p.NG;

  auto load_slab = [&](int ch, int buf) {
    float* dst = slab0 + buf * slab_sz;
    const int c0 = ch * CK;
    const int total = p.slab_rows * PCS;
    for (int i = tid; i < total; i += NT) {
      int r = i / PCS, pc = i - r * PCS;
      int c = c0 + pc * 4, f = lo + r;
      bool ok = (f >= 0) && (f < lim_rows) && (c < p.C);
      const float* src = ok ? (X + (long long)f * p.ldx + c) : X;
      cp_async16(dst + r * LD + pc * 4, src, ok ? min(16, (p.C - c) * 4) : 0);
    }
  };
  auto load_w = [&](int ch, int g, int buf) {
    float* dst = wt0 + buf * wt_sz;
    const int c0 = ch * CK;
    const int total = p.TG * BN * PCS;
    for (int i = tid; i < total; i += NT) {
      int tq = i / (BN * PCS), rem = i - tq * (BN * PCS);
      int n = rem / PCS, pc = rem - n * PCS;
      int c = c0 + pc * 4, q = g * p.TG + tq;
      bool ok = (q < p.Q) && (n0 + n < p.N) && (c < p.C);
      const float* src = ok ? (Wg + (long long)q * p.w_sq + (long long)(n0 + n) * p.ldw + c) : Wg;
      cp_async16(dst + (tq * BN + n) * LD + pc * 4, src, ok ? min(16, (p.C - c) * 4) : 0);
    }
  };

  float acc[MF][NF][4];
#pragma unroll
  for (int i = 0; i < MF; ++i)
#pragma unroll
    for (int j = 0; j < NF; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;

  load_slab(0, 0);
  load_w(0, 0, 0);
  cp_async_commit();
  __syncthreads();   // s_base visible
  int rb[MF][2];
#pragma unroll
  for (int mf = 0; mf < MF; ++mf) {
    rb[mf][0] = s_base[wm * MF * 16 + mf * 16 + gid];
    rb[mf][1] = s_base[wm * MF * 16 + mf * 16 + 8 + gid];
  }

  for (int u = 0; u < U; ++u) {
    const int ch = u / p.NG, g = u - ch * p.NG;
    if (u + 1 < U) {
      const int ch1 = (u + 1) / p.NG, g1 = (u + 1) - ch1 * p.NG;
      if (g1 == 0) load_slab(ch1, ch1 & 1);
      load_w(ch1, g1, (u + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* sl = slab0 + (ch & 1) * slab_sz;
    const float* wt = wt0 + (u & 1) * wt_sz;
    const int ntaps = min(p.TG, p.Q - g * p.TG);
    for (int tq = 0; tq < ntaps; ++tq) {
      const int toff = (p.off[g * p.TG + tq] - p.off_min) * p.P;
      for (int ks = 0; ks < p.KS; ++ks) {
        const int k0 = ks * 8 + t4;
        uint32_t a[MF][4], al[MF][4];
#pragma unroll
        for (int mf = 0; mf < MF; ++mf) {
          const float* r0 = sl + (rb[mf][0] + toff) * LD + k0;
          const float* r1 = sl + (rb[mf][1] + toff) * LD + k0;
          const float f[4] = {r0[0], r1[0], r0[4], r1[4]};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            a[mf][e] = f2tf32(f[e]);
            if (PRECISE) al[mf][e] = f2tf32(f[e] - __uint_as_float(a[mf][e]));
          }
        }
#pragma unroll
        for (int nf = 0; nf < NF; ++nf) {
          const float* wr = wt + (tq * BN + wn * NF * 8 + nf * 8 + gid) * LD + k0;
          const float g0 = wr[0], g1 = wr[4];
          uint32_t bb[2] = {f2tf32(g0), f2tf32(g1)};
          if (PRECISE) {
            uint32_t bl[2] = {f2tf32(g0 - __uint_as_float(bb[0])), f2tf32(g1 - __uint_as_float(bb[1]))};
#pragma unroll
            for (int mf = 0; mf < MF; ++mf) {
              mma_tf32(acc[mf][nf], al[mf], bb);
              mma_tf32(acc[mf][nf], a[mf], bl);
            }
          }
#pragma unroll
          for (int mf = 0; mf < MF; ++mf) mma_tf32(acc[mf][nf], a[mf], bb);
        }
      }
    }
    __syncthreads();
  }

  // ---- epilogue
  float* Y = p.y + b * p.y_sb + h * p.y_sh;
  const float* R = p.res ? (p.res + b * p.r_sb + h * p.r_sh) : nullptr;
  const int olen = p.out_len ? p.out_len[b] : 0x7fffffff;
#pragma unroll
  for (int mf = 0; mf < MF; ++mf) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int m = wm * MF * 16 + mf * 16 + hf * 8 + gid;
      const int pos = p0 + m;
      if (pos >= npos) continue;
      const int j = pos / p.P, w = pos - j * p.P;
      const int oj = p.o0 + j * p.os;
      const long long orow = (long long)oj * p.P + w;
      const bool live = oj < olen;
#pragma unroll
      for (int nf = 0; nf < NF; ++nf) {
        const int n = n0 + wn * NF * 8 + nf * 8 + 2 * t4;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (n + e < p.N) {
            float v = acc[mf][nf][hf * 2 + e];
            if (p.bias) v += p.bias[h * p.b_sh + n + e];
            if (R) v += R[orow * p.ldr + n + e];
            v = apply_act(v, p.act, p.slope);
            Y[orow * p.ldy + n + e] = live ? v : 0.f;
          }
        }
      }
    }
  }
}

// ============================================================================================
// W kernel (weight gradient): dW[q][n][c] += sum_pos Yg[orow][n] * X[irow(pos,q)][c]
// GEMM view: M = n (out channels), N = (q, c) columns (taps folded into the column space so that skinny layers
// fill the tile), K = positions (split over CTAs and K warps; each writes a partial, ordered_sum adds them in order).
// ============================================================================================
template <int TN, int TC, int WARPS_N, int WARPS_C, int WARPS_K, bool PRECISE>
__global__ void __launch_bounds__(NT) gconv_w_kernel(const __grid_constant__ GP p) {
  static_assert(WARPS_N * WARPS_C * WARPS_K * 32 == NT, "8 warps");
  constexpr int MF = TN / (WARPS_N * 16), NF = TC / (WARPS_C * 8);
  static_assert(MF >= 1 && NF >= 1, "tile");
  constexpr int RK = (WARPS_K * 8 > 32) ? WARPS_K * 8 : 32;   // positions per pipeline stage
  constexpr int LDA = TN + 8, LDB = TC + 8;    // == 8 (mod 32) -> conflict-free fragment reads
  extern __shared__ __align__(16) float wsm[];
  float (*As)[RK][LDA] = reinterpret_cast<float (*)[RK][LDA]>(wsm);                     // [2][RK][LDA]
  float (*Bs)[RK][LDB] = reinterpret_cast<float (*)[RK][LDB]>(wsm + 2 * RK * LDA);      // [2][RK][LDB]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gid = lane >> 2, t4 = lane & 3;
  const int wk = warp % WARPS_K, wc = (warp / WARPS_K) % WARPS_C, wnn = warp / (WARPS_K * WARPS_C);
  const int z = p.zoff + blockIdx.z;
  const int b = z / p.H, h = z - b * p.H;
  const int Cq = (p.C + 3) & ~3;                      // per-tap column pitch (16-byte pieces never straddle taps)
  const int ncols = p.Q * Cq;
  const int tiles_c = (ncols + TC - 1) / TC;
  const int tn = blockIdx.y / tiles_c, tc = blockIdx.y - tn * tiles_c;
  const int n0 = tn * TN, col0 = tc * TC;
  const float* X = p.x + b * p.x_sb + h * p.x_sh;
  const float* Yg = p.y + b * p.y_sb + h * p.y_sh;
  const int npos = p.J * p.P;
  const int pbeg = blockIdx.x * p.rch, pend = min(npos, pbeg + p.rch);
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);

  auto load_stage = [&](int r0, int buf) {
    constexpr int PA = TN / 4, PB = TC / 4;
    for (int i = tid; i < RK * PA; i += NT) {
      int rr = i / PA, pc = i - rr * PA;
      int pos = r0 + rr, n = n0 + pc * 4;
      bool ok = (pos < pend) && (n < p.N);
      const float* src = Yg;
      if (ok) {
        int j = pos / p.P, w = pos - j * p.P;
        long long orow = (long long)(p.o0 + j * p.os) * p.P + w;
        src = Yg + orow * p.ldy + n;
      }
      cp_async16(&As[buf][rr][pc * 4], src, ok ? min(16, (p.N - n) * 4) : 0);
    }
    for (int i = tid; i < RK * PB; i += NT) {
      int rr = i / PB, pc = i - rr * PB;
      int pos = r0 + rr, col = col0 + pc * 4;
      int q = col / Cq, c = col - q * Cq;
      bool ok = (pos < pend) && (q < p.Q) && (c < p.C);
      const float* src = X;
      if (ok) {
        int j = pos / p.P, w = pos - j * p.P;
        int ij = j * p.is + p.off[q];
        ok = (ij >= 0) && (ij < lim);
        if (ok) src = X + ((long long)ij * p.P + w) * p.ldx + c;
      }
      cp_async16(&Bs[buf][rr][pc * 4], src, ok ? min(16, (p.C - c) * 4) : 0);
    }
  };

  float acc[MF][NF][4];
#pragma unroll
  for (int i = 0; i < MF; ++i)
#pragma unroll
    for (int j = 0; j < NF; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;

  const int nst = (pend - pbeg + RK - 1) / RK;
  if (nst > 0) {
    load_stage(pbeg, 0);
    cp_async_commit();
  }
  for (int s = 0; s < nst; ++s) {
    if (s + 1 < nst) {
      load_stage(pbeg + (s + 1) * RK, (s + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int buf = s & 1;
#pragma unroll
    for (int ks = 0; ks < RK / 8; ++ks) {
      if ((ks % WARPS_K) != wk) continue;
      const int k0 = ks * 8 + t4;
      uint32_t a[MF][4], al[MF][4];
#pragma unroll
      for (int mf = 0; mf < MF; ++mf) {
        const int nb = wnn * MF * 16 + mf * 16 + gid;
        const float f[4] = {As[buf][k0][nb], As[buf][k0][nb + 8], As[buf][k0 + 4][nb], As[buf][k0 + 4][nb + 8]};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          a[mf][e] = f2tf32(f[e]);
          if (PRECISE) al[mf][e] = f2tf32(f[e] - __uint_as_float(a[mf][e]));
        }
      }
#pragma unroll
      for (int nf = 0; nf < NF; ++nf) {
        const int cb = wc * NF * 8 + nf * 8 + gid;
        const float g0 = Bs[buf][k0][cb], g1 = Bs[buf][k0 + 4][cb];
        uint32_t bb[2] = {f2tf32(g0), f2tf32(g1)};
        if (PRECISE) {
          uint32_t bl[2] = {f2tf32(g0 - __uint_as_float(bb[0])), f2tf32(g1 - __uint_as_float(bb[1]))};
#pragma unroll
          for (int mf = 0; mf < MF; ++mf) {
            mma_tf32(acc[mf][nf], al[mf], bb);
            mma_tf32(acc[mf][nf], a[mf], bl);
          }
        }
#pragma unroll
        for (int mf = 0; mf < MF; ++mf) mma_tf32(acc[mf][nf], a[mf], bb);
      }
    }
    __syncthreads();
  }

  float* Wd = p.part + (((long long)blockIdx.z * gridDim.x + blockIdx.x) * WARPS_K + wk) * ((long long)p.Q * p.N * p.C);
#pragma unroll
  for (int nf = 0; nf < NF; ++nf)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = col0 + wc * NF * 8 + nf * 8 + 2 * t4 + e;
      const int q = col / Cq, c = col - q * Cq;
      if (q >= p.Q || c >= p.C) continue;
      float* wq = Wd + (long long)q * p.N * p.C + c;
#pragma unroll
      for (int mf = 0; mf < MF; ++mf)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int n = n0 + wnn * MF * 16 + mf * 16 + hf * 8 + gid;
          if (n < p.N) wq[(long long)n * p.C] = acc[mf][nf][hf * 2 + e];
        }
    }
}

// ============================================================================================
// host side
// ============================================================================================
int g_precise = 0;          // 3xTF32 products on the mma.sync kernels (parity tests)
int g_backend_tc = 1;       // use the TMA / wgmma kernels for eligible (stride-1) launches
int gconv_tc_try(const evk_gconv_desc* d, cudaStream_t st);
int gemm_tma_try(const evk_gconv_desc* d, cudaStream_t st);

static int fill_gp(const evk_gconv_desc* d, GP& p) {
  EVK_REQUIRE(d != nullptr, EVK_ERR_ARG, "gconv: null descriptor");
  EVK_REQUIRE(d->Q >= 1 && d->Q <= EVK_MAX_TAPS, EVK_ERR_ARG, "gconv: Q=%d out of range", d->Q);
  EVK_REQUIRE(d->Z >= 1 && d->H >= 1 && d->C >= 1 && d->N >= 1 && d->J >= 0 && d->P >= 1, EVK_ERR_ARG,
              "gconv: bad sizes Z=%d H=%d C=%d N=%d J=%d P=%d", d->Z, d->H, d->C, d->N, d->J, d->P);
  EVK_REQUIRE(d->is >= 1 && d->os >= 1, EVK_ERR_ARG, "gconv: strides must be >= 1");
  p.x = d->x; p.w = d->w; p.y = d->y; p.res = d->res; p.bias = d->bias;
  p.in_len = d->in_len; p.out_len = d->out_len;
  p.x_sb = d->x_sb; p.x_sh = d->x_sh; p.w_sb = d->w_sb; p.w_sh = d->w_sh; p.w_sq = d->w_sq;
  p.y_sb = d->y_sb; p.y_sh = d->y_sh; p.r_sb = d->r_sb; p.r_sh = d->r_sh;
  p.ldx = d->ldx; p.ldw = d->ldw; p.ldy = d->ldy; p.ldr = d->ldr; p.b_sh = d->b_sh;
  p.Z = d->Z; p.H = d->H; p.C = d->C; p.N = d->N; p.Q = d->Q; p.Tin = d->Tin; p.J = d->J; p.P = d->P;
  p.is = d->is; p.os = d->os; p.o0 = d->o0; p.Tout = d->Tout; p.act = d->act; p.slope = d->slope;
  int mn = d->off[0], mx = d->off[0];
  for (int i = 0; i < d->Q; ++i) { p.off[i] = d->off[i]; mn = min(mn, d->off[i]); mx = max(mx, d->off[i]); }
  for (int i = d->Q; i < EVK_MAX_TAPS; ++i) p.off[i] = 0;
  p.off_min = mn; p.off_max = mx;
  if (d->J > 0) {
    long long last = (long long)d->o0 + (long long)(d->J - 1) * d->os;
    EVK_REQUIRE(d->o0 >= 0 && last < d->Tout, EVK_ERR_ARG, "gconv: output positions exceed Tout (o0=%d J=%d os=%d Tout=%d)",
                d->o0, d->J, d->os, d->Tout);
  }
  return EVK_OK;
}

static int check_mma_alignment(const evk_gconv_desc* d, const char* who) {
  EVK_REQUIRE(d->G <= 1, EVK_ERR_UNSUPPORTED, "%s: pass groups as the inner batch (H = groups), not G", who);
  EVK_REQUIRE((d->ldx % 4) == 0 && (d->ldw % 4) == 0 && (d->w_sq % 4) == 0, EVK_ERR_ARG,
              "%s: ldx, ldw, w_sq must be multiples of 4 (ldx=%d ldw=%d)", who, d->ldx, d->ldw);
  EVK_REQUIRE((d->x_sb % 4) == 0 && (d->x_sh % 4) == 0 && (d->w_sb % 4) == 0 && (d->w_sh % 4) == 0, EVK_ERR_ARG,
              "%s: batch strides must be multiples of 4", who);
  EVK_REQUIRE(((uintptr_t)d->x % 16) == 0 && ((uintptr_t)d->w % 16) == 0, EVK_ERR_ARG, "%s: x/w must be 16-byte aligned", who);
  return EVK_OK;
}

template <int WARPS_M, int WARPS_N, int MF, int NF, bool PRECISE>
static int launch_f(GP& p, cudaStream_t st) {
  constexpr int BN = WARPS_N * NF * 8;
  // stage shape: K per stage ~ 64..128
  int KS, TG;
  if (p.Q == 1) KS = 8;
  else if (p.Q <= 3) KS = 4;
  else if (p.Q <= 7) KS = 2;
  else KS = 1;
  while (KS > 1 && (KS * 8) / 2 >= p.C) KS >>= 1;     // do not over-chunk tiny C
  int NG = (p.Q + 7) / 8;
  TG = (p.Q + NG - 1) / NG;
  NG = (p.Q + TG - 1) / TG;
  const int jspan = min(p.J > 0 ? p.J - 1 : 0, (BM + p.P - 2) / p.P);
  auto smem_for = [&](int ks) {
    int CK = ks * 8, LD = CK + 4;
    long long slab_rows = ((long long)jspan * p.is + (p.off_max - p.off_min)) * p.P + p.P;
    return (long long)(2 * slab_rows * LD + 2 * (long long)TG * BN * LD) * 4;
  };
  while (KS > 1 && smem_for(KS) > 200 * 1024) KS >>= 1;
  long long smem = smem_for(KS);
  EVK_REQUIRE(smem <= 220 * 1024, EVK_ERR_UNSUPPORTED,
              "gconv_fwd: slab too large (%lld B; is=%d P=%d span=%d)", smem, p.is, p.P, p.off_max - p.off_min);
  p.KS = KS; p.TG = TG; p.NG = NG;
  p.slab_rows = (int)(((long long)jspan * p.is + (p.off_max - p.off_min)) * p.P + p.P);
  auto kern = gconv_f_kernel<WARPS_M, WARPS_N, MF, NF, PRECISE>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    attr_set = true;
  }
  dim3 grid(cdiv((long long)p.J * p.P, BM), cdiv(p.N, BN), p.Z);
  if (grid.x == 0) return EVK_OK;
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "gconv_fwd: grid too large");
  kern<<<grid, NT, (size_t)smem, st>>>(p);
  return check_launch("gconv_f_kernel");
}

}  // namespace evk

using namespace evk;

extern "C" int evk_set_precise(int32_t on) { g_precise = on ? 1 : 0; return EVK_OK; }
extern "C" int evk_get_precise(void) { return g_precise; }
extern "C" int evk_set_backend(int32_t tensor_core) { g_backend_tc = tensor_core ? 1 : 0; return EVK_OK; }

extern "C" int evk_gconv_fwd(const evk_gconv_desc* d, evk_stream_t stream) {
  GP p;
  int rc = fill_gp(d, p);
  if (rc) return rc;
  rc = check_mma_alignment(d, "gconv_fwd");
  if (rc) return rc;
  EVK_REQUIRE(d->y != nullptr && d->x != nullptr && d->w != nullptr, EVK_ERR_ARG, "gconv_fwd: null tensor");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_backend_tc && !g_precise && (d->ldx % 4) == 0) {
    rc = gemm_tma_try(d, st);          // TMA-fed persistent wgmma GEMM / implicit-GEMM conv
    if (rc <= 0) { if (rc == 0) g_disp_flops[0] += desc_flops(d); return rc; }
    EVK_REQUIRE(!(d->drop_rng && d->drop_p > 0.f), EVK_ERR_UNSUPPORTED, "gconv_fwd: fused dropout needs a launch the TMA kernel takes");
    rc = gconv_tc_try(d, st);
    if (rc <= 0) { if (rc == 0) g_disp_flops[1] += desc_flops(d); return rc; }
  }
  EVK_REQUIRE(!(d->drop_rng && d->drop_p > 0.f), EVK_ERR_UNSUPPORTED, "gconv_fwd: fused dropout needs a launch the TMA kernel takes");
  g_disp_flops[2] += desc_flops(d);
  // pick the N tile with the least padding (prefer wide)
  const int N = p.N;
  auto waste = [&](int bn) { return (long long)cdiv(N, bn) * bn; };
  int best = 128;
  long long bw = waste(128);
  const int cands[4] = {64, 32, 16, 8};
  for (int i = 0; i < 4; ++i) {
    long long w = waste(cands[i]);
    if (w < bw) { bw = w; best = cands[i]; }
  }
#define EVK_F(WM, WN, MF_, NF_) (g_precise ? launch_f<WM, WN, MF_, NF_, true>(p, st) : launch_f<WM, WN, MF_, NF_, false>(p, st))
  switch (best) {
    case 128: return EVK_F(4, 2, 2, 8);
    case 64: return EVK_F(4, 2, 2, 4);
    case 32: return EVK_F(8, 1, 1, 4);
    case 16: return EVK_F(8, 1, 1, 2);
    default: return EVK_F(8, 1, 1, 1);
  }
#undef EVK_F
}

// W[b'][h'][q][n][c] += sum over the batch items b of [b0, b0 + nb) (all of them when w_sb == 0, else b = b') and the groups h
// (all when w_sh == 0, else h = h') and the S1 partials j, in that nesting order, of part[((b - b0) * H + h) * S1 + j][q][n][c]
__global__ void gconv_w_sum_kernel(const GP p, int b0, int nb, int S1) {
  const long long nwt = (long long)p.Q * p.N * p.C;
  const int Bo = p.w_sb == 0 ? 1 : nb, Ho = p.w_sh == 0 ? 1 : p.H;
  const long long total = (long long)Bo * Ho * nwt;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i % nwt, bh = i / nwt;
    const int hh = (int)(bh % Ho), bb = (int)(bh / Ho);
    const int c = (int)(e % p.C), n = (int)((e / p.C) % p.N), q = (int)(e / ((long long)p.C * p.N));
    float acc = 0.f;
    for (int b = (p.w_sb == 0 ? 0 : bb); b < (p.w_sb == 0 ? nb : bb + 1); ++b)
      for (int h = (p.w_sh == 0 ? 0 : hh); h < (p.w_sh == 0 ? p.H : hh + 1); ++h)
        for (int j = 0; j < S1; ++j) acc += p.part[(((long long)b * p.H + h) * S1 + j) * nwt + e];
    p.w[(long long)(b0 + bb) * p.w_sb + (long long)hh * p.w_sh + (long long)q * p.w_sq + (long long)n * p.ldw + c] += acc;
  }
}

template <int TN, int TC, int WN, int WC, int WK, bool PRECISE>
static int launch_w(GP& p, cudaStream_t st) {
  constexpr int RK = (WK * 8 > 32) ? WK * 8 : 32;
  constexpr size_t smem = (size_t)2 * RK * ((TN + 8) + (TC + 8)) * sizeof(float);
  const long long npos = (long long)p.J * p.P;
  const int Cq = (p.C + 3) & ~3;
  const int tiles = cdiv(p.N, TN) * cdiv((long long)p.Q * Cq, TC);
  // aim for >= ~4 waves of the SMs, but keep >= 256 positions per CTA
  long long ctas_fixed = (long long)tiles * p.Z;
  long long want = ((long long)kNumSMs * 8 + ctas_fixed - 1) / ctas_fixed;
  long long rch = (npos + want - 1) / want;
  rch = ((rch + 31) / 32) * 32;
  if (rch < 256) rch = 256;
  // partials: [batch items of one launch][H][S1 = chunks * WK][Q][N][C], at most PART_CAP floats per launch
  constexpr long long PART_CAP = 40ll << 20;            // floats of partials per launch (batch slices beyond it)
  if (npos == 0 || p.Z == 0) return EVK_OK;
  const long long nwt = (long long)p.Q * p.N * p.C;
  const int B = p.Z / p.H;
  while (rch < npos && (long long)cdiv(npos, rch) * p.H * WK * nwt > PART_CAP) rch *= 2;
  p.rch = (int)rch;
  const int S1 = cdiv(npos, rch) * WK;
  const int nb = (int)max(1ll, min((long long)B, PART_CAP / ((long long)S1 * p.H * nwt)));
  Scratch part_buf((long long)nb * p.H * S1 * nwt, st);
  p.part = part_buf.p;
  EVK_REQUIRE(p.part, EVK_ERR_CUDA, "gconv_wgrad: scratch allocation failed");
  dim3 grid(cdiv(npos, rch), tiles, nb * p.H);
  if (grid.x == 0) return EVK_OK;
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "gconv_wgrad: grid too large");
  auto kern = gconv_w_kernel<TN, TC, WN, WC, WK, PRECISE>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr_set = true;
  }
  for (int b0 = 0; b0 < B; b0 += nb) {                             // batch slices in order, each reduced before the next
    const int n_b = min(nb, B - b0);
    p.zoff = b0 * p.H;
    grid.z = n_b * p.H;
    kern<<<grid, NT, smem, st>>>(p);
    if (int rc = check_launch("gconv_w_kernel")) return rc;
    const long long total = (long long)(p.w_sb == 0 ? 1 : n_b) * (p.w_sh == 0 ? 1 : p.H) * nwt;
    gconv_w_sum_kernel<<<(unsigned)min((long long)kNumSMs * 16, (total + 255) / 256), 256, 0, st>>>(p, b0, n_b, S1);
    if (int rc = check_launch("gconv_w_sum")) return rc;
  }
  return EVK_OK;
}

extern "C" int evk_gconv_wgrad(const evk_gconv_desc* d, evk_stream_t stream) {
  GP p;
  int rc = fill_gp(d, p);
  if (rc) return rc;
  EVK_REQUIRE(d->G <= 1, EVK_ERR_UNSUPPORTED, "gconv_wgrad: pass groups as the inner batch (H = groups), not G");
  EVK_REQUIRE((d->ldx % 4) == 0 && (d->ldy % 4) == 0, EVK_ERR_ARG,
              "gconv_wgrad: ldx, ldy must be multiples of 4 (ldx=%d ldy=%d)", d->ldx, d->ldy);
  EVK_REQUIRE(((uintptr_t)d->x % 16) == 0 && ((uintptr_t)d->y % 16) == 0, EVK_ERR_ARG, "gconv_wgrad: x/y must be 16-byte aligned");
  EVK_REQUIRE((d->x_sb % 4) == 0 && (d->x_sh % 4) == 0 && (d->y_sb % 4) == 0 && (d->y_sh % 4) == 0, EVK_ERR_ARG,
              "gconv_wgrad: batch strides must be multiples of 4");
  EVK_REQUIRE(d->y != nullptr && d->x != nullptr && d->w != nullptr, EVK_ERR_ARG, "gconv_wgrad: null tensor");
  cudaStream_t st = (cudaStream_t)stream;
  g_disp_flops[5] += desc_flops(d);
  const long long ncols = (long long)p.Q * ((p.C + 3) & ~3);
#define EVK_W(...) (g_precise ? launch_w<__VA_ARGS__, true>(p, st) : launch_w<__VA_ARGS__, false>(p, st))
  if (p.N <= 16) {
    if (ncols <= 16) return EVK_W(16, 16, 1, 1, 8);
    return EVK_W(16, 64, 1, 4, 2);
  }
  if (ncols <= 16) return EVK_W(64, 16, 4, 1, 2);
  if (p.N <= 32) return EVK_W(32, 64, 2, 4, 1);
  if (p.N >= 128 && ncols >= 128) return EVK_W(128, 128, 2, 4, 1);
  return EVK_W(64, 64, 2, 4, 1);
#undef EVK_W
}
