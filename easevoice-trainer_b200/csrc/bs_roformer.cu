// BS-Roformer separation (uvr5/bs_roformer.py, lib_v5/vr_network/bs_roformer.py:327-553), inference only:
//   rope_attn_fwd_kernel  the axial Attention from the packed QKV + gate GEMM output to just before to_out: rotary embedding of
//                         q and k, softmax(q k^T / 8) v, times sigmoid(gate) per head.  Sequences are described by strides, so
//                         the time and the frequency transformers read the same [B, T, bands, dim] activations.
//   band_input_kernel     the STFT output in the band-split operand layout 'b t (f s c)', each band's segment L2-normalised
//   row_l2norm_kernel     x / max(||x||, 1e-12) per row (every other RMSNorm; gamma * sqrt(dim) is folded into the next Linear)
// The attention follows bert.cu: CTA = 64 queries of one (sequence, head), four warps of 16 rows, 32-key tiles through a
// cp.async double buffer with an online softmax; TF32 mma.sync m16n8k8 with fp32 accumulation (3xTF32 under
// evk_set_precise(1)).  No atomics: every output is summed in one fixed order.
#include "flash_common.cuh"

namespace evk {
namespace {

constexpr int HD = 64;       // head dim
constexpr int BQ = 64;       // queries per CTA (4 warps x 16 rows)
constexpr int BK = 32;       // keys per tile
constexpr int LDK = 68;      // smem row pitch in floats: conflict-free for the K (row gq, col t) and V (row 2t, col gq) reads

struct RopeArgs {
  const float* qkv; int ld;      // row = [q (H*64) | k (H*64) | v (H*64) | gate logits (H)]
  float* o; int ldo;             // row = [h*64 + d]
  const float2* cs;              // [L][32] (cos, sin) of p * theta_i
  int L, H, nqt, inner;
  long long s_outer, s_inner, s_tok;   // in rows: sequence n = (n / inner, n % inner) starts at row
                                       // (n / inner) * s_outer + (n % inner) * s_inner, token t at + t * s_tok
  float sl2;
};

// stage a [BK x 64] tile of tokens r0.. (zero-filled past L) into smem with pitch LDK: 128 threads, 4 x 16 B each
__device__ __forceinline__ void stage_tok(float* s, const float* g, long long rowstep, int r0, int L) {
#pragma unroll
  for (int c = threadIdx.x; c < BK * 16; c += 128) {
    const int r = c >> 4, q4 = (c & 15) * 4, row = r0 + r;
    cp_async16(s + r * LDK + q4, g + (row < L ? row : 0) * rowstep + q4, row < L ? 16 : 0);
  }
}

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

// interleaved rotation of element c of a row x at position pos: out[2i] = x[2i] cos - x[2i+1] sin, out[2i+1] = x[2i+1] cos + x[2i] sin
__device__ __forceinline__ float rope1(const float* x, int c, float2 cs) {
  const float a = x[c], b = x[c ^ 1];
  return (c & 1) ? a * cs.x + b * cs.y : a * cs.x - b * cs.y;
}

template <bool PR>
__global__ void __launch_bounds__(128) rope_attn_fwd_kernel(RopeArgs a) {
  __shared__ __align__(16) float sK[2][BK * LDK];
  __shared__ __align__(16) float sV[2][BK * LDK];
  const int seq = blockIdx.x / a.nqt, i0 = (blockIdx.x - seq * a.nqt) * BQ, h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L, D = a.H * HD;
  const long long base = (long long)(seq / a.inner) * a.s_outer + (long long)(seq % a.inner) * a.s_inner;
  const long long step = a.s_tok * a.ld;                     // floats between consecutive tokens
  const float* Q = a.qkv + base * a.ld + h * HD;
  const float* K = Q + D;
  const float* V = Q + 2 * D;

  // rotated Q fragments (16 rows x 64 per warp), split once; rows past L read as zero
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  uint32_t qh[8][4], ql[8][4];
  {
    const float* qa = Q + (ra < L ? ra : 0) * step;
    const float* qb = Q + (rb < L ? rb : 0) * step;
    const float2* ca = a.cs + (ra < L ? ra : 0) * 32;
    const float2* cb = a.cs + (rb < L ? rb : 0) * 32;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int c0 = ks * 8 + t, c1 = c0 + 4;
      const float x[4] = {ra < L ? rope1(qa, c0, ca[c0 >> 1]) : 0.f, rb < L ? rope1(qb, c0, cb[c0 >> 1]) : 0.f,
                          ra < L ? rope1(qa, c1, ca[c1 >> 1]) : 0.f, rb < L ? rope1(qb, c1, cb[c1 >> 1]) : 0.f};
      split4<PR>(x, qh[ks], ql[ks]);
    }
  }

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;

  const int nkt = (L + BK - 1) / BK;
  stage_tok(sK[0], K, step, 0, L);
  stage_tok(sV[0], V, step, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nkt; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nkt) {
      stage_tok(sK[cur ^ 1], K, step, (kt + 1) * BK, L);
      stage_tok(sV[cur ^ 1], V, step, (kt + 1) * BK, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    float* Ks = sK[cur];
    const float* Vs = sV[cur];
    const int j0 = kt * BK;
    // rotate the K tile in place: 32 rows x 32 pairs, 8 pairs per thread
#pragma unroll
    for (int e = threadIdx.x; e < BK * 32; e += 128) {
      const int r = e >> 5, i = e & 31;
      if (j0 + r < L) {
        const float2 cs = a.cs[(j0 + r) * 32 + i];
        float2* p = reinterpret_cast<float2*>(Ks + r * LDK + 2 * i);
        const float2 x = *p;
        *p = make_float2(x.x * cs.x - x.y * cs.y, x.y * cs.x + x.x * cs.y);
      }
    }
    __syncthreads();
    // S[16 x 32] = Q K^T
    float s[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        mma_p<PR>(s[nt], qh[ks], ql[ks], Ks[(nt * 8 + gq) * LDK + ks * 8 + t], Ks[(nt * 8 + gq) * LDK + ks * 8 + t + 4]);
    }
    const bool full = j0 + BK <= L;                          // CTA-uniform: only the last tile carries keys past L
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int j = j0 + nt * 8 + 2 * t;
      const bool ok0 = full || j < L, ok1 = full || j + 1 < L;
      s[nt][0] = ok0 ? s[nt][0] * a.sl2 : -INFINITY;
      s[nt][1] = ok1 ? s[nt][1] * a.sl2 : -INFINITY;
      s[nt][2] = ok0 ? s[nt][2] * a.sl2 : -INFINITY;
      s[nt][3] = ok1 ? s[nt][3] * a.sl2 : -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // key 0 is always present (L >= 1), so mx is finite from the first tile on
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
  const long long ostep = a.s_tok * a.ldo;
  float* O = a.o + base * a.ldo + h * HD;
  const float* G = a.qkv + base * a.ld + 3 * D + h;
  // sigmoid(gate) / l: l >= 1, the row maximum contributes ex2(0)
  const float ga = ra < L ? 1.f / ((1.f + expf(-G[ra * step])) * l0) : 0.f;
  const float gb = rb < L ? 1.f / ((1.f + expf(-G[rb * step])) * l1) : 0.f;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    if (ra < L) *reinterpret_cast<float2*>(O + ra * ostep + n * 8 + 2 * t) = make_float2(acc[n][0] * ga, acc[n][1] * ga);
    if (rb < L) *reinterpret_cast<float2*>(O + rb * ostep + n * 8 + 2 * t) = make_float2(acc[n][2] * gb, acc[n][3] * gb);
  }
}

// One CTA per (b, t): gather the row 'b t (f s c)' from cplx [(b S + s) T + t][NB][2] into shared memory, then one warp per band
// divides the band's segment [2 S bo[i], 2 S bo[i+1]) by max(||segment||, 1e-12)
__global__ void __launch_bounds__(256) band_input_kernel(const float2* __restrict__ cplx, int S, int T, int NB,
                                                         const int* __restrict__ bo, int nb, float* __restrict__ y, int ldy) {
  extern __shared__ float srow[];
  const int bt = blockIdx.x, b = bt / T, t = bt - b * T;
  for (int e = threadIdx.x; e < S * NB; e += blockDim.x) {
    const int f = e / S, s = e - f * S;
    const float2 v = cplx[((long long)(b * S + s) * T + t) * NB + f];
    srow[2 * e] = v.x;
    srow[2 * e + 1] = v.y;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float* yr = y + (long long)bt * ldy;
  for (int i = warp; i < nb; i += nw) {
    const int c0 = 2 * S * bo[i], c1 = 2 * S * bo[i + 1];
    float ss = 0.f;
    for (int c = c0 + lane; c < c1; c += 32) ss += srow[c] * srow[c];
    const float den = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    for (int c = c0 + lane; c < c1; c += 32) yr[c] = srow[c] / den;
  }
}

// one warp per row: y = x / max(||x||, 1e-12)
__global__ void __launch_bounds__(256) row_l2norm_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy,
                                                         long long rows, int C) {
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* xr = x + r * ldx;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) ss += xr[c] * xr[c];
  const float den = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  float* yr = y + r * ldy;
  for (int c = lane; c < C; c += 32) yr[c] = xr[c] / den;
}

}  // namespace
extern int g_precise;
}  // namespace evk

using namespace evk;

extern "C" int evk_rope_attn_fwd(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                                 int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok,
                                 evk_stream_t stream) {
  EVK_REQUIRE(qkvg && cs && o, EVK_ERR_ARG, "rope_attn: null tensor");
  EVK_REQUIRE(H > 0 && H <= 65535 && L > 0 && n_outer > 0 && n_inner > 0 && s_tok > 0 && s_outer >= 0 && s_inner >= 0, EVK_ERR_ARG,
              "rope_attn: bad sizes H=%d L=%d outer=%d inner=%d", H, L, n_outer, n_inner);
  EVK_REQUIRE(ld % 4 == 0 && ldo % 2 == 0 && ld >= 3 * H * HD + H && ldo >= H * HD, EVK_ERR_ARG,
              "rope_attn: row pitches must hold the packed row (ld %% 4 == 0, ldo %% 2 == 0)");
  EVK_REQUIRE((uintptr_t)qkvg % 16 == 0 && (uintptr_t)o % 8 == 0 && (uintptr_t)cs % 8 == 0, EVK_ERR_ARG,
              "rope_attn: qkvg must be 16-byte and o, cs 8-byte aligned");
  const int nqt = cdiv(L, BQ);
  const long long blocks = (long long)n_outer * n_inner * nqt;
  EVK_REQUIRE(blocks <= 0x7fffffff, EVK_ERR_ARG, "rope_attn: too many sequences");
  RopeArgs a{qkvg, ld, o, ldo, reinterpret_cast<const float2*>(cs), L, H, nqt, n_inner, s_outer, s_inner, s_tok,
             0.125f * LOG2E};
  dim3 grid((unsigned)blocks, H);
  cudaStream_t st = (cudaStream_t)stream;
  if (g_precise) rope_attn_fwd_kernel<true><<<grid, 128, 0, st>>>(a);
  else rope_attn_fwd_kernel<false><<<grid, 128, 0, st>>>(a);
  return check_launch("rope_attn_fwd");
}

extern "C" int evk_bs_band_input(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, const int32_t* band_off,
                                 int32_t n_bands, float* y, int32_t ldy, evk_stream_t stream) {
  EVK_REQUIRE(cplx && band_off && y, EVK_ERR_ARG, "bs_band_input: null tensor");
  EVK_REQUIRE(B > 0 && (S == 1 || S == 2) && T > 0 && n_bins > 0 && n_bands > 0 && ldy >= 2 * S * n_bins, EVK_ERR_ARG,
              "bs_band_input: bad sizes B=%d S=%d T=%d bins=%d ldy=%d", B, S, T, n_bins, ldy);
  const size_t smem = (size_t)2 * S * n_bins * sizeof(float);
  EVK_REQUIRE(smem <= 48 * 1024, EVK_ERR_UNSUPPORTED, "bs_band_input: %d bins x %d channels do not fit shared memory", n_bins, S);
  EVK_REQUIRE((long long)B * T <= 0x7fffffff, EVK_ERR_ARG, "bs_band_input: too many frames");
  band_input_kernel<<<(unsigned)(B * T), 256, smem, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(cplx), S, T, n_bins,
                                                                              band_off, n_bands, y, ldy);
  return check_launch("bs_band_input");
}

extern "C" int evk_row_l2norm(const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && y && C > 0 && rows >= 0 && ldx >= C && ldy >= C, EVK_ERR_ARG, "row_l2norm: bad arguments");
  if (rows == 0) return EVK_OK;
  EVK_REQUIRE((rows + 7) / 8 <= 0x7fffffff, EVK_ERR_ARG, "row_l2norm: too many rows");
  row_l2norm_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, ldx, y, ldy, rows, C);
  return check_launch("row_l2norm");
}
