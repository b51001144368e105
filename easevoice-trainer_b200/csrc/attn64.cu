// Fused attention of head dim 64, inference only, for two callers:
//   evk_attn_pad_fwd   the BERT text encoder (transformers BertSelfAttention with an attention_mask that is a prefix of ones):
//                      O = softmax(Q K^T * scale + mask) V per (batch, head), key j visible to every query iff j < lens[b]
//   evk_rope_attn_fwd  the BS-Roformer axial Attention (uvr5/bs_roformer.py, lib_v5/vr_network/bs_roformer.py:327-553) from
//                      the packed QKV + gate GEMM output to just before to_out: rotary embedding of q and k,
//                      softmax(q k^T / 8) v, times sigmoid(gate) per head
// Both launch attn64_fwd_kernel; its ROPE parameter selects the rotary embedding, the gate and "every key is visible".
// evk_rope_attn_fwd_h16 is the Roformer attention with fp16 / bf16 operands on m16n8k16 (rope_attn_h16_kernel); it shares
// the tile staging, the rotation, the softmax step and the output store with attn64_fwd_kernel.
// Sequences are described by strides, so the Roformer's time and frequency transformers read the same [B, T, bands, dim]
// activations.  The [L, L] scores never exist: CTA = 64 queries of one (sequence, head) (four warps of 16 rows), streaming
// 32-key tiles through a cp.async double buffer with an online softmax; only the ceil(len / 32) tiles that hold a visible key
// are read.  TF32 mma.sync m16n8k8 with fp32 accumulation (3xTF32 under evk_set_precise(1)), the operand conventions of
// attn_mma.cuh.  No atomics: every output is summed in one fixed order.
#include "attn_mma.cuh"

namespace evk {
namespace {

constexpr int HD = 64;       // head dim
constexpr int BQ = 64;       // queries per CTA (4 warps x 16 rows)
constexpr int BK = 32;       // keys per tile
constexpr int LDK = 68;      // smem row pitch in floats: conflict-free for the K (row gq, col t) and V (row 2t, col gq) reads

struct Attn64Args {
  const float *q, *k, *v; int ld;      // token rows; head h at columns h*64.. of q, k and v
  const float* gate;                   // ROPE: gate logit of head h at column h of a token row
  float* o; int ldo;                   // row = [h*64 + d]
  const float2* cs;                    // ROPE: [L][32] (cos, sin) of p * theta_i
  const long long* lens;               // !ROPE: keys j < clamp(lens[n], 1, L) of sequence n are visible (ROPE: all L)
  int L, nqt, inner;
  long long s_outer, s_inner, s_tok;   // in rows: sequence n = (n / inner, n % inner) starts at row
                                       // (n / inner) * s_outer + (n % inner) * s_inner, token t at + t * s_tok
  float scale;
};

// element c of rope_pair on the pair of a row x that holds c, computed alone
__device__ __forceinline__ float rope1(const float* x, int c, float2 cs) {
  const float a = x[c], b = x[c ^ 1];
  return (c & 1) ? a * cs.x + b * cs.y : a * cs.x - b * cs.y;
}

// One key tile's online-softmax step for the warp's rows g and g + 8, in fp32: the scores s of keys j0 .. j0 + 31 are scaled
// by sl2 (scale * log2 e; keys at or past len masked), the running maxima m and sums l updated, acc rescaled, and s replaced
// by the tile's probabilities ex2(s - m)
__device__ __forceinline__ void softmax_tile(float (&s)[4][4], float (&acc)[8][4], float& m0, float& m1, float& l0, float& l1,
                                             int j0, int len, float sl2) {
  const int t = threadIdx.x & 3;
  const bool full = j0 + BK <= len;                          // CTA-uniform: only the last tile carries keys at or past len
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
  const float c0 = ex2(m0 - mx0), c1 = ex2(m1 - mx1);        // m == -inf on the first tile -> 0
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
}

// The warp's rows ra, rb (those below L) of acc / l to o, times sigmoid(gate logit) under ROPE
template <bool ROPE>
__device__ __forceinline__ void store_rows(const Attn64Args& a, long long base, int h, int ra, int rb, const float (&acc)[8][4],
                                           float l0, float l1) {
  const int t = threadIdx.x & 3, L = a.L;
  const long long step = a.s_tok * a.ld;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // 1 / l, times sigmoid(gate) under ROPE: l >= 1, the row maximum contributes ex2(0)
  float ga, gb;
  if (ROPE) {
    const float* G = a.gate + base * a.ld + h;
    ga = ra < L ? 1.f / ((1.f + expf(-G[ra * step])) * l0) : 0.f;
    gb = rb < L ? 1.f / ((1.f + expf(-G[rb * step])) * l1) : 0.f;
  } else {
    ga = 1.f / l0;
    gb = 1.f / l1;
  }
  const long long ostep = a.s_tok * a.ldo;
  float* O = a.o + base * a.ldo + h * HD;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    if (ra < L) *reinterpret_cast<float2*>(O + ra * ostep + n * 8 + 2 * t) = make_float2(acc[n][0] * ga, acc[n][1] * ga);
    if (rb < L) *reinterpret_cast<float2*>(O + rb * ostep + n * 8 + 2 * t) = make_float2(acc[n][2] * gb, acc[n][3] * gb);
  }
}

template <bool PR, bool ROPE>
__global__ void __launch_bounds__(128) attn64_fwd_kernel(Attn64Args a) {
  __shared__ __align__(16) float sK[2][BK * LDK];
  __shared__ __align__(16) float sV[2][BK * LDK];
  const int seq = blockIdx.x / a.nqt, i0 = (blockIdx.x - seq * a.nqt) * BQ, h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L;
  const int len = ROPE ? L : (int)min(max(a.lens[seq], 1ll), (long long)L);   // CTA-uniform: keys j < len are visible
  const long long base = (long long)(seq / a.inner) * a.s_outer + (long long)(seq % a.inner) * a.s_inner;
  const long long step = a.s_tok * a.ld;                     // floats between consecutive tokens
  const float* Q = a.q + base * a.ld + h * HD;
  const float* K = a.k + base * a.ld + h * HD;
  const float* V = a.v + base * a.ld + h * HD;
  const float sl2 = a.scale * LOG2E;

  // Q fragments (16 rows x 64 per warp), rotated (ROPE) and split once; rows past L read as zero
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  uint32_t qh[8][4], ql[8][4];
  {
    const float* qa = Q + (ra < L ? ra : 0) * step;
    const float* qb = Q + (rb < L ? rb : 0) * step;
    const float2* ca = ROPE ? a.cs + (ra < L ? ra : 0) * 32 : nullptr;
    const float2* cb = ROPE ? a.cs + (rb < L ? rb : 0) * 32 : nullptr;
    auto qx = [](const float* x, const float2* cs, int c) { return ROPE ? rope1(x, c, cs[c >> 1]) : x[c]; };
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int c0 = ks * 8 + t, c1 = c0 + 4;
      const float x[4] = {ra < L ? qx(qa, ca, c0) : 0.f, rb < L ? qx(qb, cb, c0) : 0.f,
                          ra < L ? qx(qa, ca, c1) : 0.f, rb < L ? qx(qb, cb, c1) : 0.f};
      split4<PR>(x, qh[ks], ql[ks]);
    }
  }

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;

  const int nkt = (len + BK - 1) / BK;
  stage_tile<BK, HD, LDK>(sK[0], K, step, 0, L);
  stage_tile<BK, HD, LDK>(sV[0], V, step, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nkt; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nkt) {
      stage_tile<BK, HD, LDK>(sK[cur ^ 1], K, step, (kt + 1) * BK, L);
      stage_tile<BK, HD, LDK>(sV[cur ^ 1], V, step, (kt + 1) * BK, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    float* Ks = sK[cur];
    const int j0 = kt * BK;
    if (ROPE) {
      // rotate the K tile in place: 32 rows x 32 pairs, 8 pairs per thread
#pragma unroll
      for (int e = threadIdx.x; e < BK * 32; e += 128) {
        const int r = e >> 5, i = e & 31;
        if (j0 + r < L) {
          float2* p = reinterpret_cast<float2*>(Ks + r * LDK + 2 * i);
          *p = rope_pair(*p, a.cs[(j0 + r) * 32 + i]);
        }
      }
      __syncthreads();
    }
    float s[4][4];
    gemm_nt<PR, 4, 8, LDK>(s, qh, ql, Ks);                   // S[16 x 32] = Q K^T
    softmax_tile(s, acc, m0, m1, l0, l1, j0, len, sl2);
    gemm_pn<PR, 4, 8, LDK>(acc, s, sV[cur]);                 // acc[16 x 64] += P[16 x 32] V[32 x 64]
    __syncthreads();
  }
  store_rows<ROPE>(a, base, h, ra, rb, acc, l0, l1);
}

// evk_rope_attn_fwd_h16: the rotary gated attention with 16-bit operands (fp16, or bf16 when BF16).  The same CTA, staging
// and softmax as attn64_fwd_kernel<PR, true>; q, k (rotated in fp32) and v are rounded to 16 bits, the scores come from
// m16n8k16 with fp32 accumulation, and P is rounded to 16 bits for P V.  Each staged fp32 K / V tile is converted once into
// 16-bit tiles that all four warps read with ldmatrix.
constexpr int LDH = 72;      // 16-bit tile pitch in elements: 144-byte rows, conflict-free ldmatrix
template <bool BF16>
__global__ void __launch_bounds__(128) rope_attn_h16_kernel(Attn64Args a) {
  __shared__ __align__(16) float sK[2][BK * LDK];
  __shared__ __align__(16) float sV[2][BK * LDK];
  __shared__ __align__(16) uint16_t hK[BK * LDH], hV[BK * LDH];
  const int seq = blockIdx.x / a.nqt, i0 = (blockIdx.x - seq * a.nqt) * BQ, h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L;
  const long long base = (long long)(seq / a.inner) * a.s_outer + (long long)(seq % a.inner) * a.s_inner;
  const long long step = a.s_tok * a.ld;                     // floats between consecutive tokens
  const float* Q = a.q + base * a.ld + h * HD;
  const float* K = a.k + base * a.ld + h * HD;
  const float* V = a.v + base * a.ld + h * HD;
  const float sl2 = a.scale * LOG2E;

  // Q fragments (16 rows x 64 per warp) of k-steps ks: columns 16 ks + 2t, +1 and 16 ks + 2t + 8, +9 are rotary pairs
  // 8 ks + t and 8 ks + t + 4; rows past L are zeros
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  uint32_t qf[4][4];
  {
    const float* qa = Q + (ra < L ? ra : 0) * step;
    const float* qb = Q + (rb < L ? rb : 0) * step;
    const float2* ca = a.cs + (ra < L ? ra : 0) * 32;
    const float2* cb = a.cs + (rb < L ? rb : 0) * 32;
    auto q2 = [](bool ok, const float* x, const float2* cs, int i) {
      const float2 r = ok ? rope_pair(*reinterpret_cast<const float2*>(x + 2 * i), cs[i]) : make_float2(0.f, 0.f);
      return to_h16x2<BF16>(r.x, r.y);
    };
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int i = ks * 8 + t;
      qf[ks][0] = q2(ra < L, qa, ca, i);
      qf[ks][1] = q2(rb < L, qb, cb, i);
      qf[ks][2] = q2(ra < L, qa, ca, i + 4);
      qf[ks][3] = q2(rb < L, qb, cb, i + 4);
    }
  }

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;

  const int nkt = (L + BK - 1) / BK;
  stage_tile<BK, HD, LDK>(sK[0], K, step, 0, L);
  stage_tile<BK, HD, LDK>(sV[0], V, step, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nkt; ++kt) {
    const int cur = kt & 1, j0 = kt * BK;
    if (kt + 1 < nkt) {
      stage_tile<BK, HD, LDK>(sK[cur ^ 1], K, step, j0 + BK, L);
      stage_tile<BK, HD, LDK>(sV[cur ^ 1], V, step, j0 + BK, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();                                         // tile kt staged; every warp is done with tile kt - 1's hK, hV
    tile_h16<BF16, true, BK, LDK, LDH>(hK, sK[cur], a.cs, j0, L);
    tile_h16<BF16, false, BK, LDK, LDH>(hV, sV[cur], nullptr, j0, L);
    // hK, hV written; sK[cur], sV[cur] read, so the next iteration's prefetch into them (after this barrier) is safe
    __syncthreads();
    float s[4][4];
    gemm_nt_h16<BF16, 4, LDH>(s, qf, hK);                    // S[16 x 32] = h(Q) h(K)^T
    softmax_tile(s, acc, m0, m1, l0, l1, j0, L, sl2);
    gemm_pn_h16<BF16, 2, 8, LDH>(acc, s, hV);               // acc[16 x 64] += h(P)[16 x 32] h(V)[32 x 64]
  }
  store_rows<true>(a, base, h, ra, rb, acc, l0, l1);
}

}  // namespace
extern int g_precise;

template <bool ROPE>
static int attn64_fwd(const Attn64Args& a, dim3 grid, cudaStream_t st, const char* what) {
  if (g_precise) attn64_fwd_kernel<true, ROPE><<<grid, 128, 0, st>>>(a);
  else attn64_fwd_kernel<false, ROPE><<<grid, 128, 0, st>>>(a);
  return check_launch(what);
}

}  // namespace evk

using namespace evk;

extern "C" int evk_attn_pad_fwd(const float* q, const float* k, const float* v, int32_t ld, float* o, int32_t ldo, int32_t B,
                                int32_t H, int32_t L, const int64_t* lens, float scale, cudaStream_t st) {
  EVK_REQUIRE(q && k && v && o && lens, EVK_ERR_ARG, "attn_pad: null tensor");
  EVK_REQUIRE(B > 0 && H > 0 && L > 0 && H <= 65535 && (long long)B * cdiv(L, BQ) <= 0x7fffffff, EVK_ERR_ARG,
              "attn_pad: bad sizes B=%d H=%d L=%d", B, H, L);
  EVK_REQUIRE(ld % 4 == 0 && ldo % 2 == 0 && ld >= HD && ldo >= HD, EVK_ERR_ARG,
              "attn_pad: row pitches must be multiples of 4 (ld) / 2 (ldo) floats");
  EVK_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) % 16 == 0 && (uintptr_t)o % 8 == 0, EVK_ERR_ARG,
              "attn_pad: q/k/v must be 16-byte and o 8-byte aligned");
  const int nqt = cdiv(L, BQ);
  // B sequences of L tokens, sequence b at row b * L
  Attn64Args a{q, k, v, ld, nullptr, o, ldo, nullptr, (const long long*)lens, L, nqt, 1, L, 0, 1, scale};
  return attn64_fwd<false>(a, dim3(B * nqt, H), st, "attn_pad_fwd");
}

// The checks and launch geometry of evk_rope_attn_fwd and evk_rope_attn_fwd_h16
static int rope_attn_args(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                          int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok, Attn64Args& a,
                          dim3& grid) {
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
  // row = [q (H*64) | k (H*64) | v (H*64) | gate logits (H)]
  const int D = H * HD;
  a = Attn64Args{qkvg, qkvg + D, qkvg + 2 * D, ld, qkvg + 3 * D, o, ldo, reinterpret_cast<const float2*>(cs), nullptr, L, nqt,
                 n_inner, s_outer, s_inner, s_tok, 0.125f};
  grid = dim3((unsigned)blocks, H);
  return EVK_OK;
}

extern "C" int evk_rope_attn_fwd(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                                 int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok,
                                 evk_stream_t stream) {
  Attn64Args a;
  dim3 grid;
  const int rc = rope_attn_args(qkvg, ld, cs, o, ldo, H, L, n_outer, s_outer, n_inner, s_inner, s_tok, a, grid);
  if (rc) return rc;
  return attn64_fwd<true>(a, grid, (cudaStream_t)stream, "rope_attn_fwd");
}

extern "C" int evk_rope_attn_fwd_h16(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                                     int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok,
                                     int32_t bf16, evk_stream_t stream) {
  Attn64Args a;
  dim3 grid;
  const int rc = rope_attn_args(qkvg, ld, cs, o, ldo, H, L, n_outer, s_outer, n_inner, s_inner, s_tok, a, grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (bf16) rope_attn_h16_kernel<true><<<grid, 128, 0, st>>>(a);
  else rope_attn_h16_kernel<false><<<grid, 128, 0, st>>>(a);
  return check_launch("rope_attn_fwd_h16");
}
