// Fused bidirectional attention with per-row key lengths for the BERT text encoder (transformers BertSelfAttention with an
// attention_mask that is a prefix of ones):
//   O = softmax(Q K^T * scale + mask) V     per (batch, head), head dim 64, key j visible to every query iff j < lens[b]
// Inference only.  The [B*H, L, L] scores never exist: CTA = 64 queries of one (b, h) (four warps of 16 rows), streaming
// 32-key tiles through a cp.async double buffer with an online softmax; only the ceil(lens[b] / 32) tiles that hold a
// visible key are read.  TF32 mma.sync m16n8k8 with fp32 accumulation, the operand conventions of flash.cu: the S
// accumulator fragment is reused as the A fragment of P.V by permuting the contraction index (k = t <-> key 2t,
// k = t + 4 <-> key 2t + 1).  No atomics: every output is summed in one fixed order.
#include "flash_common.cuh"

namespace evk {
namespace {

constexpr int HD = 64;       // head dim
constexpr int BQ = 64;       // queries per CTA (4 warps x 16 rows)
constexpr int BK = 32;       // keys per tile
constexpr int LDK = 68;      // smem row pitch in floats: conflict-free for the K (row gq, col t) and V (row 2t, col gq) reads

struct PadArgs {
  const float *q, *k, *v;
  int ld;
  float* o; int ldo;
  int L;
  const long long* lens;
  float scale;
};

// stage a [BK x 64] tile (rows r0.., zero-filled past L) into smem with pitch LDK: 128 threads, 4 x 16 B each
__device__ __forceinline__ void stage_kv(float* s, const float* g, int ld, int r0, int L) {
#pragma unroll
  for (int c = threadIdx.x; c < BK * 16; c += 128) {
    const int r = c >> 4, q4 = (c & 15) * 4, row = r0 + r;
    cp_async16(s + r * LDK + q4, g + (size_t)(row < L ? row : 0) * ld + q4, row < L ? 16 : 0);
  }
}

// 3xTF32 split (PR): x = hi + lo, a*b ~ hi*hi + lo*hi + hi*lo.  Otherwise the B operand (K / V rows from shared memory) goes
// in as raw fp32 bits (the tensor core truncates the low mantissa bits) and the A operands are rounded to nearest.
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
    uint32_t bh[2] = {__float_as_uint(b0), __float_as_uint(b1)};
    mma_tf32(c, ah, bh);
  }
}

template <bool PR>
__global__ void __launch_bounds__(128) attn_pad_fwd_kernel(PadArgs a) {
  __shared__ __align__(16) float sK[2][BK * LDK];
  __shared__ __align__(16) float sV[2][BK * LDK];
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L;
  const int len = (int)min(max(a.lens[b], 1ll), (long long)L);
  const size_t boff = (size_t)b * L * a.ld + (size_t)h * HD;
  const float *Q = a.q + boff, *K = a.k + boff, *V = a.v + boff;
  const float sl2 = a.scale * LOG2E;

  // Q fragments (16 rows x 64 per warp), split once; rows past L read as zero
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  uint32_t qh[8][4], ql[8][4];
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const float x[4] = {ra < L ? Q[(size_t)ra * a.ld + ks * 8 + t] : 0.f, rb < L ? Q[(size_t)rb * a.ld + ks * 8 + t] : 0.f,
                        ra < L ? Q[(size_t)ra * a.ld + ks * 8 + t + 4] : 0.f, rb < L ? Q[(size_t)rb * a.ld + ks * 8 + t + 4] : 0.f};
    split4<PR>(x, qh[ks], ql[ks]);
  }

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;

  const int nkt = (len + BK - 1) / BK;
  stage_kv(sK[0], K, a.ld, 0, L);
  stage_kv(sV[0], V, a.ld, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nkt; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nkt) {
      stage_kv(sK[cur ^ 1], K, a.ld, (kt + 1) * BK, L);
      stage_kv(sV[cur ^ 1], V, a.ld, (kt + 1) * BK, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const float* Ks = sK[cur];
    const float* Vs = sV[cur];
    // S[16 x 32] = Q K^T
    float s[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        mma_p<PR>(s[nt], qh[ks], ql[ks], Ks[(nt * 8 + gq) * LDK + ks * 8 + t], Ks[(nt * 8 + gq) * LDK + ks * 8 + t + 4]);
    }
    const int j0 = kt * BK;
    const bool full = j0 + BK <= len;                        // CTA-uniform: only the last tile carries masked keys
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int j = j0 + nt * 8 + 2 * t;
      const bool ok0 = full || j < len, ok1 = full || j + 1 < len;
      s[nt][0] = ok0 ? s[nt][0] * sl2 : -INFINITY;
      s[nt][1] = ok1 ? s[nt][1] * sl2 : -INFINITY;
      s[nt][2] = ok0 ? s[nt][2] * sl2 : -INFINITY;
      s[nt][3] = ok1 ? s[nt][3] * sl2 : -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // key 0 is always visible (len >= 1), so mx is finite from the first tile on
    const float c0 = ex2(m0 - mx0), c1 = ex2(m1 - mx1);      // m == -inf on the first tile -> 0
    m0 = mx0; m1 = mx1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = ex2(s[nt][0] - mx0); s[nt][1] = ex2(s[nt][1] - mx0);
      s[nt][2] = ex2(s[nt][2] - mx1); s[nt][3] = ex2(s[nt][3] - mx1);
      rs0 += s[nt][0] + s[nt][1]; rs1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
#pragma unroll
    for (int n = 0; n < 8; ++n) { acc[n][0] *= c0; acc[n][1] *= c0; acc[n][2] *= c1; acc[n][3] *= c1; }
    // acc[16 x 64] += P[16 x 32] V[32 x 64]
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      const float p[4] = {s[kb][0], s[kb][2], s[kb][1], s[kb][3]};
      uint32_t ph[4], pl[4];
      split4<PR>(p, ph, pl);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
        mma_p<PR>(acc[nt], ph, pl, Vs[(kb * 8 + 2 * t) * LDK + nt * 8 + gq], Vs[(kb * 8 + 2 * t + 1) * LDK + nt * 8 + gq]);
    }
    __syncthreads();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0v = 1.f / l0, i1v = 1.f / l1;                 // l >= 1: the row maximum contributes ex2(0)
  float* O = a.o + (size_t)b * L * a.ldo + (size_t)h * HD;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    if (ra < L) *reinterpret_cast<float2*>(O + (size_t)ra * a.ldo + n * 8 + 2 * t) = make_float2(acc[n][0] * i0v, acc[n][1] * i0v);
    if (rb < L) *reinterpret_cast<float2*>(O + (size_t)rb * a.ldo + n * 8 + 2 * t) = make_float2(acc[n][2] * i1v, acc[n][3] * i1v);
  }
}

}  // namespace
extern int g_precise;
}  // namespace evk

using namespace evk;

extern "C" int evk_attn_pad_fwd(const float* q, const float* k, const float* v, int32_t ld, float* o, int32_t ldo, int32_t B,
                                int32_t H, int32_t L, const int64_t* lens, float scale, cudaStream_t st) {
  EVK_REQUIRE(q && k && v && o && lens, EVK_ERR_ARG, "attn_pad: null tensor");
  EVK_REQUIRE(B > 0 && H > 0 && L > 0 && L <= 512 && B <= 65535 && H <= 65535, EVK_ERR_ARG,
              "attn_pad: bad sizes B=%d H=%d L=%d (1 <= L <= 512)", B, H, L);
  EVK_REQUIRE(ld % 4 == 0 && ldo % 2 == 0 && ld >= HD && ldo >= HD, EVK_ERR_ARG,
              "attn_pad: row pitches must be multiples of 4 (ld) / 2 (ldo) floats");
  EVK_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) % 16 == 0 && (uintptr_t)o % 8 == 0, EVK_ERR_ARG,
              "attn_pad: q/k/v must be 16-byte and o 8-byte aligned");
  PadArgs a{q, k, v, ld, o, ldo, L, (const long long*)lens, scale};
  dim3 grid(cdiv(L, BQ), H, B);
  if (g_precise) attn_pad_fwd_kernel<true><<<grid, 128, 0, st>>>(a);
  else attn_pad_fwd_kernel<false><<<grid, 128, 0, st>>>(a);
  return check_launch("attn_pad_fwd");
}
