// Common device/host helpers for libevk_sm90.so (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/evk.h"

namespace evk {

// ---- thread-local error string (evk_last_error) -------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> EVK_ERR_CUDA

#define EVK_REQUIRE(cond, code, ...)        \
  do {                                      \
    if (!(cond)) {                          \
      evk::set_error(__VA_ARGS__);          \
      return (code);                        \
    }                                       \
  } while (0)

// dispatch accounting slots (evk_dispatch_stats)
extern double g_disp_flops[EVK_DISPATCH_SLOTS];
static inline double desc_flops(const evk_gconv_desc* d) {
  return 2.0 * d->Z * (double)d->J * d->P * d->N * (d->C / (d->G > 0 ? d->G : 1)) * d->Q;
}

// ---- generalised 1-D convolution (evk_gconv_desc) -----------------------------------------------
// The descriptor's operand fields as a kernel parameter block.  The mma.sync, wgmma and direct conv kernels each derive
// their own parameters from it and add only their tuning fields.
struct ConvP {
  const float* x; float* w; float* y; const float* res; const float* bias;
  const int* in_len; const int* out_len;
  long long x_sb, x_sh, w_sb, w_sh, w_sq, y_sb, y_sh, r_sb, r_sh;
  int ldx, ldw, ldy, ldr, b_sh;
  int Z, H, C, N, Q, Tin, J, P, is, os, o0, Tout, act;
  float slope;
  int off_min, off_max;        // extremes of off[0, Q)
  int off[EVK_MAX_TAPS];       // off[Q, EVK_MAX_TAPS) = 0
  int G;                       // groups, >= 1 (the direct kernels; the tensor-core kernels take groups as H)
};
// Validates d and fills p; `who` names the entry point in the error message.  Returns EVK_OK or EVK_ERR_ARG.
int conv_params(const evk_gconv_desc* d, ConvP& p, const char* who);
// The direct CUDA-core kernels (conv_direct.cu): the conv entry points run the launches they cannot tile on them.
int conv_direct_fwd(const evk_gconv_desc* d, cudaStream_t st);
int conv_direct_dgrad(const evk_gconv_desc* d, cudaStream_t st);   // d->x is written (dX), d->y read (dY)
int conv_direct_wgrad(const evk_gconv_desc* d, cudaStream_t st);

// The evk_act epilogue.
__device__ __forceinline__ float conv_act(float v, int act, float slope) {
  if (act == EVK_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == EVK_ACT_RELU) return fmaxf(v, 0.f);
  if (act == EVK_ACT_TANH) return tanhf(v);
  if (act == EVK_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

// SMs of an H100 SXM: sizes the grids of grid-stride and persistent launches (the TMA GEMM queries the device instead).
constexpr int kNumSMs = 132;

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---- deterministic cross-block sums ------------------------------------------------------------
// Float additions do not associate, so a result that many blocks add into with atomics changes in its last bits from run
// to run (and a training run amplifies that).  Kernels instead write one partial per block into library scratch and
// ordered_sum adds the partials in block order:
//   dst[o*d_so + r*d_sr + c] += sum_{s < S} part[s*ps + (o*R + r)*Cn + c]      (ps = O*R*Cn unless given)
// Scratch is stream-ordered device memory for those partials: allocated on stream st from the library's memory pool
// (cudaMallocFromPoolAsync) and freed on st (cudaFreeAsync) when it goes out of scope, after the kernels that use it have
// been enqueued.  The pool allocator orders reuse across streams itself, and under CUDA-graph capture the pair becomes the
// graph's own allocation / free nodes.  p is null when n == 0 or the allocation failed.
struct Scratch {
  float* p = nullptr;
  cudaStream_t st;
  Scratch(long long n, cudaStream_t s) : st(s) { alloc(n); }
  ~Scratch();
  void alloc(long long n);
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
};
int ordered_sum(const float* part, int S, long long ps, int O, int R, int Cn, float* dst, long long d_so, long long d_sr, cudaStream_t st);
static inline int ordered_sum(const float* part, int S, int O, int R, int Cn, float* dst, long long d_so, long long d_sr, cudaStream_t st) {
  return ordered_sum(part, S, (long long)O * R * Cn, O, R, Cn, dst, d_so, d_sr, st);
}

// ---- device helpers -----------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// 16-byte async copy global->shared; src_bytes < 16 zero-fills the remainder (0 => all zeros).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
               "r"(src_bytes));
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
               "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ uint32_t f2tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return r;
}

// D(16x8, f32) += A(16x8, tf32, row) * B(8x8, tf32, col)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// fp32 -> fp16 (BF16 false) or bf16 bits, round to nearest even
template <bool BF16>
__device__ __forceinline__ uint16_t to_h16(float v) {
  if constexpr (BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(v));
  else return __half_as_ushort(__float2half_rn(v));
}

template <bool BF16>
__device__ __forceinline__ uint32_t to_h16x2(float lo, float hi) {
  return (uint32_t)to_h16<BF16>(lo) | ((uint32_t)to_h16<BF16>(hi) << 16);
}

// d += A * B over K = 16: a0..a3 = A(g, 2t..2t+1), A(g+8, 2t..), A(g, 2t+8..), A(g+8, 2t+8..); b0, b1 = B(2t.., g), B(2t+8.., g)
// with g = lane / 4, t = lane % 4; d = (g, 2t..2t+1), (g+8, 2t..2t+1).
template <bool BF16>
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum for blockDim.x <= 1024 (result valid in all threads)
__device__ __forceinline__ float block_sum(float v, float* red /* >= 33 floats */) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// block-wide max in the order of block_sum (result valid in all threads)
__device__ __forceinline__ float block_max(float v, float* red /* >= 33 floats */) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) {
    t = warp_max(t);
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// Philox-4x32-10 counter RNG (graph-safe: state = (seed, offset) read from device memory)
struct Philox {
  uint32_t k0, k1;
  __device__ Philox(uint64_t seed) : k0((uint32_t)seed), k1((uint32_t)(seed >> 32)) {}
  __device__ uint4 operator()(uint64_t ctr, uint64_t stream) const {
    uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = (uint32_t)stream, c3 = (uint32_t)(stream >> 32);
    uint32_t a = k0, b = k1;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
      uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
      uint32_t n0 = hi1 ^ c1 ^ a, n1 = lo1, n2 = hi0 ^ c3 ^ b, n3 = lo0;
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
      a += 0x9E3779B9u; b += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
};
// Cheap counter-based dropout for FUSED kernels (GEMM epilogue, LayerNorm): one hash decides a group of 4 consecutive elements
// through four 16-bit fields (drop iff field < round(p * 65536)).  Key = Philox(seed)(offset, stream id) read from the
// device-resident RNG state, so it is CUDA-graph safe and changes every step like the stand-alone dropout kernel.
struct DropK { uint32_t k0, k1, thr; float inv; };
__device__ __forceinline__ DropK dropk_make(const unsigned long long* rng, unsigned long long sid, float p) {
  DropK d{0u, 0u, 0u, 1.f};
  if (p > 0.f) {
    Philox ph(rng[0]);
    const uint4 r = ph(rng[1], sid);
    d.k0 = r.x; d.k1 = r.y;
    d.thr = (uint32_t)fminf(p * 65536.f + 0.5f, 65535.f);
    d.inv = 1.f / (1.f - p);
  }
  return d;
}
// scale factors (0 or 1/(1-p)) of the 4 elements of group g4 (= linear element index / 4)
__device__ __forceinline__ void dropk_scale4(const DropK& d, unsigned long long g4, float (&m)[4]) {
  uint32_t x = (uint32_t)g4 * 0x9E3779B1u + d.k0;
  x ^= (uint32_t)(g4 >> 32) * 0x85EBCA77u;
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  uint32_t y = (x + d.k1) * 0x9E3779B1u;
  y ^= y >> 15;
  m[0] = (x & 0xffffu) >= d.thr ? d.inv : 0.f;
  m[1] = (x >> 16) >= d.thr ? d.inv : 0.f;
  m[2] = (y & 0xffffu) >= d.thr ? d.inv : 0.f;
  m[3] = (y >> 16) >= d.thr ? d.inv : 0.f;
}

__device__ __forceinline__ float u32_to_unit(uint32_t x) { return (x >> 8) * (1.0f / 16777216.0f); }  // [0,1)

}  // namespace evk
