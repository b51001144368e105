// Fused prefix-LM attention for the stage-1 AR GPT (t2s_model.py:456-487 mask + patched_mha_with_cache.py SDPA call):
//   O = dropout(softmax(Q K^T / sqrt(dk) + mask)) V     per (batch, head), dk == 32
// The [B*H, L, L] score / mask tensors the reference materialises (1.68 GB per layer at B=16, L=1280) never exist:
// the mask is a closed form of (prefix, x_len[b], y_len[b]), the softmax is online, the backward recomputes P from the
// saved row log-sum-exp.  Three kernels, all TF32 mma.sync m16n8k8 with fp32 accumulation:
//   flash_fwd   : CTA = 64 queries of one (b,h); streams 64-key tiles (cp.async double buffer)
//   flash_dq    : same tiling, dQ = scale * dS K
//   flash_dkv   : CTA = 64 keys of one (b,h); streams 64-query tiles; dV = Pd^T dO, dK = scale * dS^T Q
// (S is recomputed in both backward kernels: no atomics, no transposes, bit-reproducible.)
// The accumulator fragment of S is reused directly as the A fragment of the second GEMM by permuting the
// contraction index (k = t <-> column 2t, k = t+4 <-> column 2t+1) and loading the B rows in that order.
#include "flash_common.cuh"

namespace evk {
namespace {

constexpr int BT = 64;       // tile (queries or keys)
constexpr int LDT = 36;      // smem row pitch in floats: conflict-free for both fragment patterns

// Is EVERY (query i0.., key j0..) pair of a BT x BT tile visible?  Then the per-element mask (compares, selects and branches
// for every element) is skipped for the tile -- all but the tiles on the causal diagonal and on the x_len / y_len / prefix
// boundaries.
__device__ __forceinline__ bool tile_full(int i0, int j0, int X, int xl, int yl) {
  const int j1 = j0 + BT - 1;
  if (j1 < X) return j1 < xl;                                         // text keys only: visible to every query
  if (j0 >= X) return ((j1 - X) < yl) & (j1 <= i0);                   // audio keys only: every query row is >= i0 >= j1
  return false;                                                       // straddles the prefix boundary
}

// stage a [BT x 32] tile (rows r0.., zero-filled past L) into smem with pitch LDT: 128 threads, 4 x 16 B each
__device__ __forceinline__ void stage_tile(float* s, const float* g, int ld, int r0, int L) {
  for (int c = threadIdx.x; c < BT * 8; c += 128) {
    int r = c >> 3, q4 = (c & 7) * 4;
    int row = r0 + r;
    const float* src = g + (size_t)(row < L ? row : 0) * ld + q4;
    cp_async16(s + r * LDT + q4, src, row < L ? 16 : 0);
  }
}

// A fragments (16 rows x 32) for this warp straight from global memory (rows past L read as zero)
__device__ __forceinline__ void load_a_frags(float (&a)[4][4], const float* g, int ld, int r0, int L) {
  const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int ra = r0 + gq, rb = r0 + gq + 8;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    float x0 = ra < L ? g[(size_t)ra * ld + ks * 8 + t] : 0.f;
    float x1 = rb < L ? g[(size_t)rb * ld + ks * 8 + t] : 0.f;
    float x2 = ra < L ? g[(size_t)ra * ld + ks * 8 + t + 4] : 0.f;
    float x3 = rb < L ? g[(size_t)rb * ld + ks * 8 + t + 4] : 0.f;
    a[ks][0] = x0; a[ks][1] = x1; a[ks][2] = x2; a[ks][3] = x3;
  }
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

// C[16 x 64] = A[16 x 32] * T^T, T = smem tile [64 rows x 32] ("row n, channel k" -> B(k, n))
template <bool PR>
__device__ __forceinline__ void gemm_nt(float (&c)[8][4], const float (&a)[4][4], const float* T) {
  const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  uint32_t ah[4][4], al[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) split4<PR>(a[ks], ah[ks], al[ks]);
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      mma_p<PR>(c[nt], ah[ks], al[ks], T[(nt * 8 + gq) * LDT + ks * 8 + t], T[(nt * 8 + gq) * LDT + ks * 8 + t + 4]);
  }
}

// acc[16 x 32] += Pfrag[16 x 64] * T, T = smem tile [64 rows x 32] (contraction over tile rows, permuted)
template <bool PR>
__device__ __forceinline__ void gemm_pn(float (&acc)[4][4], const float (&p)[8][4], const float* T) {
  const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kb = 0; kb < 8; ++kb) {
    const float a[4] = {p[kb][0], p[kb][2], p[kb][1], p[kb][3]};
    uint32_t ah[4], al[4];
    split4<PR>(a, ah, al);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
      mma_p<PR>(acc[nt], ah, al, T[(kb * 8 + 2 * t) * LDT + nt * 8 + gq], T[(kb * 8 + 2 * t + 1) * LDT + nt * 8 + gq]);
  }
}

// number of key tiles a query tile starting at i0 can see
__device__ __forceinline__ int key_tiles(int i0, int L, int X, int yl) {
  int jend = max(X, min(i0 + BT, L));
  jend = min(jend, X + yl);
  jend = max(jend, min(X, L));
  return (jend + BT - 1) / BT;
}

// ------------------------------------------------------------------------------------------------
template <bool PR>
__global__ void __launch_bounds__(128, 5) flash_fwd_kernel(FlashArgs a) {
  __shared__ __align__(16) float sK[2][BT * LDT];
  __shared__ __align__(16) float sV[2][BT * LDT];
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * BT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L, X = a.X;
  const int xl = (int)a.xlen[b], yl = (int)a.ylen[b];
  const size_t boff = (size_t)b * L * a.ld + (size_t)h * DK;
  const float *Q = a.q + boff, *K = a.k + boff, *V = a.v + boff;
  const DropKey dkey = drop_key(a);
  const float sl2 = a.scale * LOG2E;

  float qa[4][4];
  load_a_frags(qa, Q, a.ld, i0 + warp * 16, L);
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  const uint32_t z = (uint32_t)(b * a.H + h);
  const uint32_t rha = drop_row(dkey, z * (uint32_t)L + (uint32_t)ra), rhb = drop_row(dkey, z * (uint32_t)L + (uint32_t)rb);

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;

  const int nt_keys = key_tiles(i0, L, X, yl);
  stage_tile(sK[0], K, a.ld, 0, L);
  stage_tile(sV[0], V, a.ld, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nt_keys; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nt_keys) {
      stage_tile(sK[cur ^ 1], K, a.ld, (kt + 1) * BT, L);
      stage_tile(sV[cur ^ 1], V, a.ld, (kt + 1) * BT, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    float s[8][4];
    gemm_nt<PR>(s, qa, sK[cur]);
    const int j0 = kt * BT;
    float mx0 = m0, mx1 = m1;
    const bool full = tile_full(i0, j0, X, xl, yl);              // CTA-uniform: interior tiles skip the mask arithmetic
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      bool ok0 = true, ok1 = true, ok2 = true, ok3 = true;
      if (!full) {
        const int j = j0 + nt * 8 + 2 * t;
        ok0 = allowed(ra, j, X, xl, yl); ok1 = allowed(ra, j + 1, X, xl, yl);
        ok2 = allowed(rb, j, X, xl, yl); ok3 = allowed(rb, j + 1, X, xl, yl);
      }
      s[nt][0] = ok0 ? s[nt][0] * sl2 : -INFINITY;
      s[nt][1] = ok1 ? s[nt][1] * sl2 : -INFINITY;
      s[nt][2] = ok2 ? s[nt][2] * sl2 : -INFINITY;
      s[nt][3] = ok3 ? s[nt][3] * sl2 : -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float e0 = (mx0 == -INFINITY) ? 0.f : mx0, e1 = (mx1 == -INFINITY) ? 0.f : mx1;
    const float c0 = ex2(m0 - e0), c1 = ex2(m1 - e1);      // m == -inf -> 0
    m0 = mx0; m1 = mx1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int j = j0 + nt * 8 + 2 * t;
      float p0 = ex2(s[nt][0] - e0), p1 = ex2(s[nt][1] - e0), p2 = ex2(s[nt][2] - e1), p3 = ex2(s[nt][3] - e1);
      rs0 += p0 + p1; rs1 += p2 + p3;
      if (dkey.thr) {
        bool k0, k1, k2, k3;
        drop_pair(dkey, rha, j, k0, k1);
        drop_pair(dkey, rhb, j, k2, k3);
        p0 = k0 ? p0 * dkey.inv : 0.f;
        p1 = k1 ? p1 * dkey.inv : 0.f;
        p2 = k2 ? p2 * dkey.inv : 0.f;
        p3 = k3 ? p3 * dkey.inv : 0.f;
      }
      s[nt][0] = p0; s[nt][1] = p1; s[nt][2] = p2; s[nt][3] = p3;
    }
    l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
#pragma unroll
    for (int n = 0; n < 4; ++n) { acc[n][0] *= c0; acc[n][1] *= c0; acc[n][2] *= c1; acc[n][3] *= c1; }
    gemm_pn<PR>(acc, s, sV[cur]);
    __syncthreads();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0v = l0 > 0.f ? 1.f / l0 : 0.f, i1v = l1 > 0.f ? 1.f / l1 : 0.f;
  float* O = a.o + (size_t)b * L * a.ldo + (size_t)h * DK;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    if (ra < L) *reinterpret_cast<float2*>(O + (size_t)ra * a.ldo + n * 8 + 2 * t) = make_float2(acc[n][0] * i0v, acc[n][1] * i0v);
    if (rb < L) *reinterpret_cast<float2*>(O + (size_t)rb * a.ldo + n * 8 + 2 * t) = make_float2(acc[n][2] * i1v, acc[n][3] * i1v);
  }
  if (t == 0) {
    float* lse = a.lse + (size_t)z * L;
    if (ra < L) lse[ra] = m0 + log2f(l0);
    if (rb < L) lse[rb] = m1 + log2f(l1);
  }
}

// delta[z][i] = sum_d dO[i][d] * O[i][d].  Eight lanes per (position, head) row, heads fastest: a warp reads 4 x 128 contiguous
// bytes of dO and of O with one float4 per lane (the one-warp-per-row version below spends its time on index divisions and
// five shuffle rounds per row).
__global__ void __launch_bounds__(256) flash_delta8_kernel(FlashArgs a) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long rows = (long long)a.B * a.H * a.L;
  long long r = t >> 3;
  const int q = (int)(t & 7);
  const bool valid = r < rows;
  if (!valid) r = rows - 1;
  const int h = (int)(r % a.H);
  const long long bi = r / a.H;                                        // b * L + i
  const int b = (int)(bi / a.L), i = (int)(bi - (long long)b * a.L);
  const float4 d = __ldg(reinterpret_cast<const float4*>(a.dout + bi * a.lddo + h * DK + 4 * q));
  const float4 o = __ldg(reinterpret_cast<const float4*>(a.o + bi * a.ldo + h * DK + 4 * q));
  float v = fmaf(d.x, o.x, fmaf(d.y, o.y, fmaf(d.z, o.z, d.w * o.w)));
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  if (valid && q == 0) ((float*)a.delta)[((size_t)b * a.H + h) * a.L + i] = v;
}
// general layout (rows not 16-byte aligned): one warp per row, lane = d
__global__ void flash_delta_kernel(FlashArgs a) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int rows = a.B * a.H * a.L;
  if (row >= rows) return;
  const int i = row % a.L, z = row / a.L, h = z % a.H, b = z / a.H;
  float v = a.dout[((size_t)b * a.L + i) * a.lddo + h * DK + lane] * a.o[((size_t)b * a.L + i) * a.ldo + h * DK + lane];
  v = warp_sum(v);
  if (lane == 0) ((float*)a.delta)[row] = v;
}

template <bool PR>
__global__ void __launch_bounds__(128, 3) flash_dq_kernel(FlashArgs a) {
  __shared__ __align__(16) float sK[2][BT * LDT];
  __shared__ __align__(16) float sV[2][BT * LDT];
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * BT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L, X = a.X;
  const int xl = (int)a.xlen[b], yl = (int)a.ylen[b];
  const size_t boff = (size_t)b * L * a.ld + (size_t)h * DK;
  const float *Q = a.q + boff, *K = a.k + boff, *V = a.v + boff;
  const float* dO = a.dout + (size_t)b * L * a.lddo + (size_t)h * DK;
  const DropKey dkey = drop_key(a);
  const float sl2 = a.scale * LOG2E;
  const uint32_t z = (uint32_t)(b * a.H + h);

  float qa[4][4], da[4][4];
  load_a_frags(qa, Q, a.ld, i0 + warp * 16, L);
  load_a_frags(da, dO, a.lddo, i0 + warp * 16, L);
  const int ra = i0 + warp * 16 + gq, rb = ra + 8;
  const uint32_t rha = drop_row(dkey, z * (uint32_t)L + (uint32_t)ra), rhb = drop_row(dkey, z * (uint32_t)L + (uint32_t)rb);
  const float* lse = a.lse + (size_t)z * L;
  const float* dl = a.delta + (size_t)z * L;
  const float lse0 = ra < L ? lse[ra] : 0.f, lse1 = rb < L ? lse[rb] : 0.f;
  const float d0 = ra < L ? dl[ra] : 0.f, d1 = rb < L ? dl[rb] : 0.f;

  float acc[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  const int nt_keys = key_tiles(i0, L, X, yl);
  stage_tile(sK[0], K, a.ld, 0, L);
  stage_tile(sV[0], V, a.ld, 0, L);
  cp_async_commit();
  for (int kt = 0; kt < nt_keys; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nt_keys) {
      stage_tile(sK[cur ^ 1], K, a.ld, (kt + 1) * BT, L);
      stage_tile(sV[cur ^ 1], V, a.ld, (kt + 1) * BT, L);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    float s[8][4], dp[8][4];
    gemm_nt<PR>(s, qa, sK[cur]);
    gemm_nt<PR>(dp, da, sV[cur]);
    const int j0 = kt * BT;
    const bool full = tile_full(i0, j0, X, xl, yl);              // CTA-uniform
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int j = j0 + nt * 8 + 2 * t;
      bool keep[4] = {true, true, true, true};
      if (dkey.thr) {
        drop_pair(dkey, rha, j, keep[0], keep[1]);
        drop_pair(dkey, rhb, j, keep[2], keep[3]);
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = (e < 2) ? ra : rb, jj = j + (e & 1);
        float p = ex2(s[nt][e] * sl2 - ((e < 2) ? lse0 : lse1));
        if (!full) p = allowed(i, jj, X, xl, yl) ? p : 0.f;
        float g = dp[nt][e];
        if (dkey.thr) g = keep[e] ? g * dkey.inv : 0.f;
        s[nt][e] = p * (g - ((e < 2) ? d0 : d1));
      }
    }
    gemm_pn<PR>(acc, s, sK[cur]);
    __syncthreads();
  }
  float* DQ = a.dq + (size_t)b * L * a.lddq + (size_t)h * DK;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    if (ra < L) *reinterpret_cast<float2*>(DQ + (size_t)ra * a.lddq + n * 8 + 2 * t) = make_float2(acc[n][0] * a.scale, acc[n][1] * a.scale);
    if (rb < L) *reinterpret_cast<float2*>(DQ + (size_t)rb * a.lddq + n * 8 + 2 * t) = make_float2(acc[n][2] * a.scale, acc[n][3] * a.scale);
  }
}

template <bool PR>
__global__ void __launch_bounds__(128, 3) flash_dkv_kernel(FlashArgs a) {
  __shared__ __align__(16) float sQ[2][BT * LDT];
  __shared__ __align__(16) float sD[2][BT * LDT];
  __shared__ float sL[2][BT], sDl[2][BT];
  __shared__ uint32_t sRh[2][BT];                                  // dropout hashes of the query rows of the staged tile
  const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * BT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int L = a.L, X = a.X;
  const int xl = (int)a.xlen[b], yl = (int)a.ylen[b];
  const size_t boff = (size_t)b * L * a.ld + (size_t)h * DK;
  const float *Q = a.q + boff, *K = a.k + boff, *V = a.v + boff;
  const float* dO = a.dout + (size_t)b * L * a.lddo + (size_t)h * DK;
  const DropKey dkey = drop_key(a);
  const float sl2 = a.scale * LOG2E;
  const uint32_t z = (uint32_t)(b * a.H + h);
  const float* lse = a.lse + (size_t)z * L;
  const float* dl = a.delta + (size_t)z * L;

  float ka[4][4], va[4][4];
  load_a_frags(ka, K, a.ld, j0 + warp * 16, L);
  load_a_frags(va, V, a.ld, j0 + warp * 16, L);
  const int ja = j0 + warp * 16 + gq, jb = ja + 8;
  const uint32_t cta = drop_col(dkey, ja), ctb = drop_col(dkey, jb);
  const uint32_t mula = (ja & 1) ? DROP_M2 : DROP_M1, mulb = (jb & 1) ? DROP_M2 : DROP_M1;
  float dk[4][4], dv[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    dk[n][0] = dk[n][1] = dk[n][2] = dk[n][3] = 0.f;
    dv[n][0] = dv[n][1] = dv[n][2] = dv[n][3] = 0.f;
  }
  // first query tile that can see this key tile: x keys are seen by everyone, y key j only by queries >= j
  const int qt0 = (j0 + BT <= X || j0 < X) ? 0 : j0 / BT;
  const int qt1 = (L + BT - 1) / BT;
  auto stage = [&](int buf, int qt) {
    stage_tile(sQ[buf], Q, a.ld, qt * BT, L);
    stage_tile(sD[buf], dO, a.lddo, qt * BT, L);
    if (threadIdx.x < BT) {
      int i = qt * BT + threadIdx.x;
      sL[buf][threadIdx.x] = i < L ? lse[i] : 0.f;
      sDl[buf][threadIdx.x] = i < L ? dl[i] : 0.f;
    }
    if (threadIdx.x >= BT) {                                         // 64 more threads: one query-row hash each
      const int r = threadIdx.x - BT;
      sRh[buf][r] = drop_row(dkey, z * (uint32_t)L + (uint32_t)(qt * BT + r));
    }
  };
  const bool dead = (j0 >= X + yl) && (j0 >= X);   // every key of the tile is padding: gradients are zero
  if (!dead) {
    stage(0, qt0);
    cp_async_commit();
    for (int qt = qt0; qt < qt1; ++qt) {
      const int cur = (qt - qt0) & 1;
      if (qt + 1 < qt1) stage(cur ^ 1, qt + 1);
      cp_async_commit();
      cp_async_wait<1>();
      __syncthreads();
      float s[8][4], dp[8][4];
      gemm_nt<PR>(s, ka, sQ[cur]);      // S^T[key][query]
      gemm_nt<PR>(dp, va, sD[cur]);     // dPd^T[key][query]
      const int i0 = qt * BT;
      const bool full = (i0 + BT <= L) && tile_full(i0, j0, X, xl, yl);   // CTA-uniform
      float pd[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int ile = nt * 8 + 2 * t;                              // even local query index: rows (ile, ile + 1) share a hash
        bool keep[4] = {true, true, true, true};
        if (dkey.thr) {
          const uint32_t r0 = sRh[cur][ile], r1 = sRh[cur][ile + 1];
          keep[0] = drop_one(dkey, r0, cta, mula);
          keep[1] = drop_one(dkey, r1, cta, mula);
          keep[2] = drop_one(dkey, r0, ctb, mulb);
          keep[3] = drop_one(dkey, r1, ctb, mulb);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int il = ile + (e & 1), i = i0 + il, j = (e < 2) ? ja : jb;
          float p = ex2(s[nt][e] * sl2 - sL[cur][il]);
          if (!full) p = (i < L && allowed(i, j, X, xl, yl)) ? p : 0.f;
          float g = dp[nt][e];
          float pdv = p;
          if (dkey.thr) {
            g = keep[e] ? g * dkey.inv : 0.f;
            pdv = keep[e] ? p * dkey.inv : 0.f;
          }
          pd[nt][e] = pdv;
          s[nt][e] = p * (g - sDl[cur][il]);
        }
      }
      gemm_pn<PR>(dv, pd, sD[cur]);
      gemm_pn<PR>(dk, s, sQ[cur]);
      __syncthreads();
    }
  }
  float* DK_ = a.dk + (size_t)b * L * a.lddq + (size_t)h * DK;
  float* DV_ = a.dv + (size_t)b * L * a.lddq + (size_t)h * DK;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    if (ja < L) {
      *reinterpret_cast<float2*>(DK_ + (size_t)ja * a.lddq + n * 8 + 2 * t) = make_float2(dk[n][0] * a.scale, dk[n][1] * a.scale);
      *reinterpret_cast<float2*>(DV_ + (size_t)ja * a.lddq + n * 8 + 2 * t) = make_float2(dv[n][0], dv[n][1]);
    }
    if (jb < L) {
      *reinterpret_cast<float2*>(DK_ + (size_t)jb * a.lddq + n * 8 + 2 * t) = make_float2(dk[n][2] * a.scale, dk[n][3] * a.scale);
      *reinterpret_cast<float2*>(DV_ + (size_t)jb * a.lddq + n * 8 + 2 * t) = make_float2(dv[n][2], dv[n][3]);
    }
  }
}

int check_common(int B, int H, int L, int X, int dk, int ld, int ldo) {
  EVK_REQUIRE(dk == DK, EVK_ERR_UNSUPPORTED, "flash attention: head dim %d unsupported (32 only)", dk);
  EVK_REQUIRE(B > 0 && H > 0 && L > 0 && X >= 0 && X <= L, EVK_ERR_ARG, "flash attention: bad sizes B=%d H=%d L=%d X=%d", B, H, L, X);
  EVK_REQUIRE(ld % 4 == 0 && ldo % 2 == 0, EVK_ERR_ARG, "flash attention: row pitches must be multiples of 4 floats");
  EVK_REQUIRE((long long)B * H * L < (1ll << 32), EVK_ERR_ARG, "flash attention: B*H*L too large");
  return 0;
}

}  // namespace
extern int g_precise;
}  // namespace evk

using namespace evk;

extern "C" int evk_flash_attn_fwd(const float* q, const float* k, const float* v, int ld, float* o, int ldo, float* lse, int32_t B,
                                  int32_t H, int32_t L, int32_t X, int32_t dk, const int64_t* xlen, const int64_t* ylen, float scale,
                                  float p_drop, const uint64_t* rng, uint64_t sid, cudaStream_t st) {
  if (int rc = check_common(B, H, L, X, dk, ld, ldo)) return rc;
  EVK_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) % 16 == 0 && (uintptr_t)o % 8 == 0, EVK_ERR_ARG,
              "flash attention: q/k/v must be 16-byte aligned");
  EVK_REQUIRE(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || rng), EVK_ERR_ARG, "flash attention: bad dropout");
  FlashArgs a{};
  a.q = q; a.k = k; a.v = v; a.ld = ld; a.o = o; a.ldo = ldo; a.lse = lse; a.B = B; a.H = H; a.L = L; a.X = X;
  a.xlen = (const long long*)xlen; a.ylen = (const long long*)ylen; a.scale = scale; a.p_drop = p_drop; a.rng = (const unsigned long long*)rng; a.sid = sid;
  dim3 grid(cdiv(L, BT), H, B);
  if (g_precise) flash_fwd_kernel<true><<<grid, 128, 0, st>>>(a);
  else flash_fwd_kernel<false><<<grid, 128, 0, st>>>(a);
  return check_launch("flash_fwd");
}

extern "C" int evk_flash_attn_bwd(const float* q, const float* k, const float* v, int ld, const float* o, int ldo,
                                  const float* lse, const float* dout, int lddo, float* delta, float* dq, float* dk_, float* dv,
                                  int lddq, int B, int H, int L, int X, int dk, const int64_t* xlen, const int64_t* ylen,
                                  float scale, float p_drop, const uint64_t* rng, uint64_t sid,
                                  cudaStream_t st) {
  if (int rc = check_common(B, H, L, X, dk, ld, ldo)) return rc;
  EVK_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dout) % 16 == 0 && lddo % 4 == 0 && lddq % 2 == 0, EVK_ERR_ARG,
              "flash attention bwd: operands must be 16-byte aligned");
  FlashArgs a{};
  a.q = q; a.k = k; a.v = v; a.ld = ld; a.o = (float*)o; a.ldo = ldo; a.lse = (float*)lse; a.dout = dout; a.lddo = lddo;
  a.delta = delta; a.dq = dq; a.dk = dk_; a.dv = dv; a.lddq = lddq; a.B = B; a.H = H; a.L = L; a.X = X;
  a.xlen = (const long long*)xlen; a.ylen = (const long long*)ylen; a.scale = scale; a.p_drop = p_drop; a.rng = (const unsigned long long*)rng; a.sid = sid;
  const int rows = B * H * L;
  if (ldo % 4 == 0 && ((uintptr_t)o % 16) == 0) flash_delta8_kernel<<<cdiv((long long)rows * 8, 256), 256, 0, st>>>(a);
  else flash_delta_kernel<<<cdiv(rows, 8), 256, 0, st>>>(a);
  if (int rc = check_launch("flash_delta")) return rc;
  dim3 grid(cdiv(L, BT), H, B);
  if (g_precise) flash_dq_kernel<true><<<grid, 128, 0, st>>>(a);
  else flash_dq_kernel<false><<<grid, 128, 0, st>>>(a);
  if (int rc = check_launch("flash_dq")) return rc;
  if (g_precise) flash_dkv_kernel<true><<<grid, 128, 0, st>>>(a);
  else flash_dkv_kernel<false><<<grid, 128, 0, st>>>(a);
  return check_launch("flash_dkv");
}
