// The mma.sync attention primitives of the prefix-LM (flash.cu) and head-dim-64 (attn64.cu) attention kernels: TF32 m16n8k8
// with fp32 accumulation, A operands from per-warp fragments, B operands from cp.async-staged shared-memory tiles, 128-thread
// CTAs; and the 16-bit (fp16 / bf16) m16n8k16 variants of attn64.cu's rotary kernel, whose B operands are 16-bit tiles
// converted from the staged fp32 ones.  Every operand rounding rule of those kernels lives here.
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

// Rotary embedding of the interleaved pair x = (x[2i], x[2i+1]) by cs = (cos, sin) of its angle, in fp32:
// (x[2i] cos - x[2i+1] sin, x[2i+1] cos + x[2i] sin)
__device__ __forceinline__ float2 rope_pair(float2 x, float2 cs) {
  return make_float2(x.x * cs.x - x.y * cs.y, x.y * cs.x + x.x * cs.y);
}

// ---- 16-bit (fp16 / bf16) operands: h = round to nearest even, products exact, fp32 accumulation -------------------------
// ldmatrix.x4 of four 8 x 8 16-bit matrices; lane l gives the address of row l % 8 of matrix l / 8.  Plain: lane (g, t) gets
// elements (g, 2t..2t+1) of each; TRANS: elements (2t, g) and (2t + 1, g).
template <bool TRANS>
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const uint16_t* p) {
  if constexpr (TRANS)
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
  else
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

// The staged fp32 tile src [ROWS x 64] (pitch PS floats, row r = token r0 + r) -> 16-bit dst (pitch PH elements), each
// interleaved pair rotated by its token's cs row first when ROT (rows at or past L are zeros and stay zeros).  128 threads.
template <bool BF16, bool ROT, int ROWS, int PS, int PH>
__device__ __forceinline__ void tile_h16(uint16_t* dst, const float* src, const float2* cs, int r0, int L) {
#pragma unroll
  for (int e = threadIdx.x; e < ROWS * 32; e += 128) {
    const int r = e >> 5, i = e & 31;
    float2 x = *reinterpret_cast<const float2*>(src + r * PS + 2 * i);
    if (ROT && r0 + r < L) x = rope_pair(x, cs[(r0 + r) * 32 + i]);
    *reinterpret_cast<uint32_t*>(dst + r * PH + 2 * i) = to_h16x2<BF16>(x.x, x.y);
  }
}

// C[16 x 8 NT] = A[16 x 64] T^T with A the m16n8k16 fragments a[ks] of k = 16 ks .., T = 16-bit smem tile [8 NT rows x 64]
// with pitch P ("row n, column k" -> B(k, n))
template <bool BF16, int NT, int P>
__device__ __forceinline__ void gemm_nt_h16(float (&c)[NT][4], const uint32_t (&a)[4][4], const uint16_t* T) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
#pragma unroll
    for (int kp = 0; kp < 2; ++kp) {
      uint32_t b[4];                                         // b0, b1 of k-step 2 kp, then of 2 kp + 1
      ldsm_x4<false>(b, T + (nt * 8 + (lane & 7)) * P + kp * 32 + (lane >> 3) * 8);
      mma16816<BF16>(c[nt], a[2 * kp][0], a[2 * kp][1], a[2 * kp][2], a[2 * kp][3], b[0], b[1]);
      mma16816<BF16>(c[nt], a[2 * kp + 1][0], a[2 * kp + 1][1], a[2 * kp + 1][2], a[2 * kp + 1][3], b[2], b[3]);
    }
  }
}

// acc[16 x 8 NT] += h(Pf)[16 x 16 KB] T, T = 16-bit smem tile [16 KB rows x 8 NT] with pitch P.  Pf is an accumulator
// fragment of gemm_nt_h16 (fp32), rounded to 16 bits here: n-tiles 2 kb and 2 kb + 1 are exactly the A fragment of k-step kb.
template <bool BF16, int KB, int NT, int P>
__device__ __forceinline__ void gemm_pn_h16(float (&acc)[NT][4], const float (&pf)[2 * KB][4], const uint16_t* T) {
  static_assert(NT % 2 == 0, "gemm_pn_h16: n-tiles in pairs");
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kb = 0; kb < KB; ++kb) {
    const uint32_t a0 = to_h16x2<BF16>(pf[2 * kb][0], pf[2 * kb][1]), a1 = to_h16x2<BF16>(pf[2 * kb][2], pf[2 * kb][3]);
    const uint32_t a2 = to_h16x2<BF16>(pf[2 * kb + 1][0], pf[2 * kb + 1][1]);
    const uint32_t a3 = to_h16x2<BF16>(pf[2 * kb + 1][2], pf[2 * kb + 1][3]);
#pragma unroll
    for (int np = 0; np < NT / 2; ++np) {
      uint32_t b[4];                                         // b0, b1 of n-tile 2 np, then of 2 np + 1
      ldsm_x4<true>(b, T + (kb * 16 + (lane & 15)) * P + np * 16 + (lane >> 4) * 8);
      mma16816<BF16>(acc[2 * np], a0, a1, a2, a3, b[0], b[1]);
      mma16816<BF16>(acc[2 * np + 1], a0, a1, a2, a3, b[2], b[3]);
    }
  }
}

}  // namespace
}  // namespace evk
