// The mma.sync attention primitives of the prefix-LM (flash.cu) and head-dim-64 (attn64.cu) attention kernels: TF32 m16n8k8
// with fp32 accumulation, A operands from per-warp fragments, B operands from cp.async-staged shared-memory tiles, 128-thread
// CTAs.  Every operand rounding rule of those kernels lives here.
#pragma once
#include "evk_common.cuh"

namespace evk {
namespace {

constexpr float LOG2E = 1.4426950408889634f;

// 2^x on the SFU without ex2()'s range handling (ex2.approx.ftz: 2^-22 relative error, 2^-inf = 0): the kernels evaluate it
// for every score and are issue-bound
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 3xTF32 split (PR): x = hi + lo with hi = tf32(x), lo = tf32(x - hi); a*b ~ hi*hi + lo*hi + hi*lo (fp32-level products,
// parity tests only -- evk_set_precise)
template <bool PR>
__device__ __forceinline__ void split4(const float (&x)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    hi[i] = f2tf32(x[i]);
    if (PR) lo[i] = f2tf32(x[i] - __uint_as_float(hi[i]));
  }
}
template <bool PR>
__device__ __forceinline__ void mma_p(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float b0, float b1) {
  if (PR) {
    uint32_t bh[2] = {f2tf32(b0), f2tf32(b1)};
    uint32_t bl[2] = {f2tf32(b0 - __uint_as_float(bh[0])), f2tf32(b1 - __uint_as_float(bh[1]))};
    mma_tf32(c, al, bh);
    mma_tf32(c, ah, bl);
    mma_tf32(c, ah, bh);
  } else {
    // the B operand (K / V / Q / dO tile rows from shared memory) is fed as raw fp32 bits: the tensor core ignores the low
    // 13 mantissa bits (truncation, as the TMA-fed wgmma GEMMs do); 128 of the 160 cvt.rna per key tile sat on the
    // critical path next to only 64 mma.  A operands (Q, dO, K, V fragments loaded once; P / dS) stay round-to-nearest.
    uint32_t bh[2] = {__float_as_uint(b0), __float_as_uint(b1)};
    mma_tf32(c, ah, bh);
  }
}

// stage a [ROWS x COLS] tile (rows r0.., zero-filled past L; row r at g + r * step) into smem with pitch P: 128 threads,
// 16 B each per step.  A row is 2^SH chunks of 16 B, split off with shifts: a signed division costs instructions and registers.
template <int ROWS, int COLS, int P>
__device__ __forceinline__ void stage_tile(float* s, const float* g, long long step, int r0, int L) {
  constexpr int SH = 31 - __builtin_clz(COLS / 4);
  static_assert(COLS == 4 << SH && ROWS * COLS % 512 == 0, "stage_tile: rows of 2^k x 16 B, 128 x 16 B per step");
#pragma unroll
  for (int i = 0; i < ROWS * COLS / 512; ++i) {
    const int c = threadIdx.x + 128 * i, r = c >> SH, q4 = (c & ((1 << SH) - 1)) * 4, row = r0 + r;
    cp_async16(s + r * P + q4, g + (row < L ? row : 0) * step + q4, row < L ? 16 : 0);
  }
}

// C[16 x 8 NT] = A[16 x 8 KS] T^T, A as (hi, lo) fragments from split4, T = smem tile [8 NT rows x 8 KS] with pitch P
// ("row n, column k" -> B(k, n))
template <bool PR, int NT, int KS, int P>
__device__ __forceinline__ void gemm_nt(float (&c)[NT][4], const uint32_t (&ah)[KS][4], const uint32_t (&al)[KS][4], const float* T) {
  const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
      mma_p<PR>(c[nt], ah[ks], al[ks], T[(nt * 8 + gq) * P + ks * 8 + t], T[(nt * 8 + gq) * P + ks * 8 + t + 4]);
  }
}

// acc[16 x 8 NT] += Pf[16 x 8 KB] T, T = smem tile [8 KB rows x 8 NT] with pitch P.  Pf is an accumulator fragment of C above,
// reused as the A fragment by permuting the contraction index (k = t <-> column 2t, k = t + 4 <-> column 2t + 1) and reading
// the rows of T in that order.
template <bool PR, int KB, int NT, int P>
__device__ __forceinline__ void gemm_pn(float (&acc)[NT][4], const float (&pf)[KB][4], const float* T) {
  const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kb = 0; kb < KB; ++kb) {
    const float a[4] = {pf[kb][0], pf[kb][2], pf[kb][1], pf[kb][3]};
    uint32_t ah[4], al[4];
    split4<PR>(a, ah, al);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
      mma_p<PR>(acc[nt], ah, al, T[(kb * 8 + 2 * t) * P + nt * 8 + gq], T[(kb * 8 + 2 * t + 1) * P + nt * 8 + gq]);
  }
}

}  // namespace
}  // namespace evk
