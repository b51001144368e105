// Channel LayerNorm (modules.py:19-31), with and without a fused dropout on the residual, the column sums of bias gradients
// and the per-channel instance norm of the HuBERT feature extractor.  Weight-norm + operand packing is in pack.cu.
#include "evk_common.cuh"

namespace evk {

// one warp per row; C <= 32*MAXV
constexpr int LN_MAXV = 32;   // up to 1024 channels

__global__ void layernorm_fwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ res, int ldr,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                     float* __restrict__ y, int ldy, float* __restrict__ stats, long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  float v[LN_MAXV];
  float s = 0.f;
  int nv = 0;
  for (int c = lane; c < C; c += 32, ++nv) {
    float t = x[row * ldx + c];
    if (res) t += res[row * ldr + c];
    v[nv] = t;
    s += t;
  }
  s = warp_sum(s);
  const float mean = s / (float)C;
  float q = 0.f;
  for (int i = 0; i < nv; ++i) { float d = v[i] - mean; q += d * d; }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / (float)C + eps);
  nv = 0;
  for (int c = lane; c < C; c += 32, ++nv) y[row * ldy + c] = (v[nv] - mean) * rstd * gamma[c] + beta[c];
  if (lane == 0 && stats) { stats[row * 2] = mean; stats[row * 2 + 1] = rstd; }
}

// A handful of rows (the token step of the KV-cache decode: ONE row of 512): the warp-per-row kernel above keeps 16 values per
// lane in a run-time indexed array (local memory) and ran 11 us per launch; here a whole 256-thread block takes a row.
// The block stages the row in shared memory and warp 0 takes both sums in the warp kernel's order (lane l adds channels l,
// l + 32, ... in turn, then warp_sum), so a row's bits do not depend on whether 8 or 9 rows share the launch: a decode batch
// of 9..64 rows gives each row what a batch of one gives it.
__global__ void __launch_bounds__(256) layernorm_fwd_block_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ res, int ldr,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                                  float* __restrict__ y, int ldy, float* __restrict__ stats, int C) {
  __shared__ float sv[32 * LN_MAXV];
  __shared__ float stat[2];
  const long long row = blockIdx.x;
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = threadIdx.x + 256 * i;
    float t = 0.f;
    if (c < C) {
      t = x[row * ldx + c];
      if (res) t += res[row * ldr + c];
      sv[c] = t;
    }
    v[i] = t;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += 32) s += sv[c];
    s = warp_sum(s);
    if (threadIdx.x == 0) stat[0] = s / (float)C;
  }
  __syncthreads();
  const float mean = stat[0];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = threadIdx.x + 256 * i;
    if (c < C) sv[c] = v[i] - mean;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float q = 0.f;
    for (int c = threadIdx.x; c < C; c += 32) { const float d = sv[c]; q += d * d; }
    q = warp_sum(q);
    if (threadIdx.x == 0) stat[1] = rsqrtf(q / (float)C + eps);
  }
  __syncthreads();
  const float rstd = stat[1];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = threadIdx.x + 256 * i;
    if (c < C) y[row * ldy + c] = (v[i] - mean) * rstd * gamma[c] + beta[c];
  }
  if (threadIdx.x == 0 && stats) { stats[row * 2] = mean; stats[row * 2 + 1] = rstd; }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)); dgamma += dy*xhat; dbeta += dy
__global__ void layernorm_bwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ res, int ldr,
                                     const float* __restrict__ gamma, const float* __restrict__ stats,
                                     const float* __restrict__ dy, int lddy, float* __restrict__ dx, int lddx,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C,
                                     int rows_per_block) {
  extern __shared__ float sm[];              // [2][C] partial dgamma/dbeta of this block
  float* sg = sm;
  float* sb = sm + C;
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sm[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float ag[LN_MAXV], ab[LN_MAXV];            // this lane's dgamma / dbeta sums over the warp's rows
  for (int i = 0; i < LN_MAXV; ++i) { ag[i] = 0.f; ab[i] = 0.f; }
  for (long long row = r0 + wid; row < r1; row += nw) {
    const float mean = stats[row * 2], rstd = stats[row * 2 + 1];
    float xh[LN_MAXV], gd[LN_MAXV];
    float s1 = 0.f, s2 = 0.f;
    int nv = 0;
    for (int c = lane; c < C; c += 32, ++nv) {
      float t = x[row * ldx + c];
      if (res) t += res[row * ldr + c];
      const float h = (t - mean) * rstd;
      const float d = dy[row * lddy + c];
      const float g = d * gamma[c];
      xh[nv] = h; gd[nv] = g;
      s1 += g; s2 += g * h;
      ag[nv] += d * h;
      ab[nv] += d;
    }
    s1 = warp_sum(s1) / (float)C;
    s2 = warp_sum(s2) / (float)C;
    nv = 0;
    for (int c = lane; c < C; c += 32, ++nv) dx[row * lddx + c] = rstd * (gd[nv] - s1 - xh[nv] * s2);
  }
  for (int w = 0; w < nw; ++w) {             // warps add their sums in a fixed order (reproducible)
    if (wid == w) {
      int nv = 0;
      for (int c = lane; c < C; c += 32, ++nv) { sg[c] += ag[nv]; sb[c] += ab[nv]; }
    }
    __syncthreads();
  }
  // partial of this block: dgamma[blockIdx.x][c], dbeta at the same index of its own array (ordered_sum adds the blocks)
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    dgamma[(long long)blockIdx.x * 2 * C + c] = sg[c];
    dgamma[(long long)blockIdx.x * 2 * C + C + c] = sb[c];
  }
}

// ---- LayerNorm(x + dropout(res)) with the dropout fused (stage-1 GPT: transformer.py:300-315) --------------------------
// One warp per row, float4 per lane (C % 4 == 0, C <= 2048, contiguous rows).  The dropout scale factors come from
// dropk_scale4 keyed by the float4's linear index, so the backward regenerates the identical mask.
// gamma / beta are parameter views (any 4-byte alignment: flat optimizer storage packs them back to back)
__device__ __forceinline__ float4 ld4_any(const float* __restrict__ p) { return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3)); }
constexpr int LND_MAXV = 4;            // float4 per lane: C <= 512 (the GPT's model width); fixed trip counts keep everything in registers
__global__ void __launch_bounds__(256) layernorm_drop_fwd_kernel(const float4* __restrict__ x, const float4* __restrict__ res,
                                                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                                 float p, const unsigned long long* __restrict__ rng, unsigned long long sid,
                                                                 float4* __restrict__ y, float* __restrict__ stats, long long rows, int C4) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const DropK dk = dropk_make(rng, sid, p);
  float4 v[LND_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LND_MAXV; ++i) {
    const int c = lane + 32 * i;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C4) {
      const long long g4 = row * C4 + c;
      float4 t = x[g4];
      const float4 r = res[g4];
      float m[4];
      dropk_scale4(dk, (unsigned long long)g4, m);
      t.x += r.x * m[0]; t.y += r.y * m[1]; t.z += r.z * m[2]; t.w += r.w * m[3];
      v[i] = t;
      s += t.x + t.y + t.z + t.w;
    }
  }
  s = warp_sum(s);
  const float mean = s / (float)(4 * C4);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LND_MAXV; ++i)
    if (lane + 32 * i < C4) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b * b + c * c + d * d;
    }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / (float)(4 * C4) + eps);
#pragma unroll
  for (int i = 0; i < LND_MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C4) {
      const float4 g = ld4_any(gamma + 4 * c), b = ld4_any(beta + 4 * c), t = v[i];
      y[row * C4 + c] = make_float4((t.x - mean) * rstd * g.x + b.x, (t.y - mean) * rstd * g.y + b.y, (t.z - mean) * rstd * g.z + b.z,
                                    (t.w - mean) * rstd * g.w + b.w);
    }
  }
  if (lane == 0) { stats[row * 2] = mean; stats[row * 2 + 1] = rstd; }
}

__global__ void __launch_bounds__(256) layernorm_drop_bwd_kernel(const float4* __restrict__ x, const float4* __restrict__ res,
                                                                 const float* __restrict__ gamma, const float* __restrict__ stats,
                                                                 const float4* __restrict__ dy, float p, const unsigned long long* __restrict__ rng,
                                                                 unsigned long long sid, float4* __restrict__ dx, float4* __restrict__ dres,
                                                                 float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C4,
                                                                 int rows_per_block) {
  extern __shared__ float sm[];              // [2][C] partial dgamma/dbeta of this block
  const int C = 4 * C4;
  float* sg = sm;
  float* sb = sm + C;
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sm[c] = 0.f;
  __syncthreads();
  const DropK dk = dropk_make(rng, sid, p);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float4 ag[LND_MAXV], ab[LND_MAXV];         // this warp's dgamma / dbeta partial sums over its rows (registers, flushed once)
#pragma unroll
  for (int i = 0; i < LND_MAXV; ++i) { ag[i] = make_float4(0.f, 0.f, 0.f, 0.f); ab[i] = ag[i]; }
  for (long long row = r0 + wid; row < r1; row += nw) {
    const float mean = stats[row * 2], rstd = stats[row * 2 + 1];
    float4 xh[LND_MAXV], gd[LND_MAXV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < LND_MAXV; ++i) {
      const int c = lane + 32 * i;
      xh[i] = make_float4(0.f, 0.f, 0.f, 0.f); gd[i] = xh[i];
      if (c < C4) {
        const long long g4 = row * C4 + c;
        float4 t = x[g4];
        const float4 r = res[g4];
        float m[4];
        dropk_scale4(dk, (unsigned long long)g4, m);
        t.x += r.x * m[0]; t.y += r.y * m[1]; t.z += r.z * m[2]; t.w += r.w * m[3];
        const float4 h = make_float4((t.x - mean) * rstd, (t.y - mean) * rstd, (t.z - mean) * rstd, (t.w - mean) * rstd);
        const float4 d = dy[g4], gm = ld4_any(gamma + 4 * c);
        const float4 g = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
        xh[i] = h; gd[i] = g;
        s1 += g.x + g.y + g.z + g.w;
        s2 += g.x * h.x + g.y * h.y + g.z * h.z + g.w * h.w;
        ag[i].x += d.x * h.x; ag[i].y += d.y * h.y; ag[i].z += d.z * h.z; ag[i].w += d.w * h.w;
        ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
      }
    }
    s1 = warp_sum(s1) / (float)C;
    s2 = warp_sum(s2) / (float)C;
#pragma unroll
    for (int i = 0; i < LND_MAXV; ++i) {
      const int c = lane + 32 * i;
      if (c < C4) {
        const long long g4 = row * C4 + c;
        const float4 h = xh[i], g = gd[i];
        const float4 o = make_float4(rstd * (g.x - s1 - h.x * s2), rstd * (g.y - s1 - h.y * s2), rstd * (g.z - s1 - h.z * s2),
                                     rstd * (g.w - s1 - h.w * s2));
        dx[g4] = o;
        float m[4];
        dropk_scale4(dk, (unsigned long long)g4, m);
        dres[g4] = make_float4(o.x * m[0], o.y * m[1], o.z * m[2], o.w * m[3]);
      }
    }
  }
  for (int w = 0; w < nw; ++w) {             // warps add their sums in a fixed order (reproducible)
    if (wid == w) {
#pragma unroll
      for (int i = 0; i < LND_MAXV; ++i) {
        const int c = lane + 32 * i;
        if (c < C4) {
          sg[4 * c] += ag[i].x; sg[4 * c + 1] += ag[i].y; sg[4 * c + 2] += ag[i].z; sg[4 * c + 3] += ag[i].w;
          sb[4 * c] += ab[i].x; sb[4 * c + 1] += ab[i].y; sb[4 * c + 2] += ab[i].z; sb[4 * c + 3] += ab[i].w;
        }
      }
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {      // partial of this block (ordered_sum adds the blocks)
    dgamma[(long long)blockIdx.x * 2 * C + c] = sg[c];
    dgamma[(long long)blockIdx.x * 2 * C + C + c] = sb[c];
  }
}

__global__ void colsum_kernel(const float* __restrict__ x, long long rows, int n, int ld, float* __restrict__ out,
                              int rows_per_block) {
  // blockDim = (32, 8): 32 columns x 8 row-lanes
  __shared__ float part[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  float acc = 0.f;
  if (c < n)
    for (long long r = r0 + threadIdx.y; r < r1; r += 8) acc += x[r * ld + c];
  part[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < n) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += part[k][threadIdx.x];
    out[(long long)blockIdx.y * n + c] = s;                      // partial of this row block (ordered_sum)
  }
}

__global__ void zero_kernel(float* p, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0.f;
}

// ---- per-channel normalisation over time (GroupNorm(C, C) of the HuBERT feature extractor), channels-last, forward only ------
// One CTA per (32 channels, batch item): 8 time lanes x 32 channel lanes; pass 1 accumulates shifted sums (shift = the channel's
// first sample, which keeps the one-pass variance stable on DC-heavy inputs), pass 2 normalises (+ optional exact GELU).
// With lens, item b is normalised over its first n = lens[b] frames only and frames t >= n are written as 0: the sums visit
// t = lane, lane + 8, ... < n in a fixed order, so the statistics of a row depend neither on T nor on what the padding holds.
// The split form (instnorm_part_kernel, instnorm_apply_kernel) shares the sums and the normalisation below.

// shifted sums of channel c over frames t0 + tl, t0 + tl + 8, ... < t1
__device__ __forceinline__ void instnorm_sums(const float* xb, int ldx, int c, float shift, long long t0, long long t1, int tl,
                                              float& s1, float& s2) {
  for (long long t = t0 + tl; t < t1; t += 8) { const float v = xb[t * ldx + c] - shift; s1 += v; s2 += v * v; }
}
// (scale, offset) of y = x * scale + offset from the shifted sums a, q over n frames
__device__ __forceinline__ float2 instnorm_coef(float a, float q, float n, float shift, float gamma, float beta, float eps) {
  const float md = a / n, var = fmaxf(q / n - md * md, 0.f);
  const float mean = md + shift, rstd = rsqrtf(var + eps), g = gamma * rstd, bb = beta - mean * g;
  return make_float2(g, bb);
}
__device__ __forceinline__ float instnorm_apply(float x, float2 gb, int act_gelu) {
  float v = x * gb.x + gb.y;
  if (act_gelu) v = 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

__global__ void __launch_bounds__(256) instnorm_cl_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float eps, int act_gelu, float* __restrict__ y,
                                                          int ldy, int T, int C, const int* __restrict__ lens) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), tl = threadIdx.x >> 5, b = blockIdx.y;
  const float* xb = x + (long long)b * T * ldx;
  float* yb = y + (long long)b * T * ldy;
  const int n = lens ? min(max(lens[b], 0), T) : T;
  const bool ok = c < C;
  const float shift = ok ? xb[c] : 0.f;
  float s1 = 0.f, s2 = 0.f;
  if (ok) instnorm_sums(xb, ldx, c, shift, 0, n, tl, s1, s2);
  __shared__ float sh1[8][32], sh2[8][32];
  sh1[tl][threadIdx.x & 31] = s1; sh2[tl][threadIdx.x & 31] = s2;
  __syncthreads();
  float a = 0.f, q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { a += sh1[i][threadIdx.x & 31]; q += sh2[i][threadIdx.x & 31]; }
  if (!ok) return;
  const float2 gb = instnorm_coef(a, q, (float)n, shift, gamma[c], beta[c], eps);
  for (int t = tl; t < n; t += 8) yb[(long long)t * ldy + c] = instnorm_apply(xb[(long long)t * ldx + c], gb, act_gelu);
  for (int t = n + tl; t < T; t += 8) yb[(long long)t * ldy + c] = 0.f;
}

// Split statistics over a plane of T pixels: CTA (32 channels, chunk, item) sums pixels [chunk * per, min(T, (chunk + 1) * per))
// as instnorm_cl_kernel does (same shift: the item's first pixel) and writes part[chunk][b][{s1, s2}][c]; ordered_sum adds the
// chunks in chunk order.  `per` depends on T only, so an item's statistics do not depend on B.
constexpr long long INORM_PER = 2048;
__global__ void __launch_bounds__(256) instnorm_part_kernel(const float* __restrict__ x, int ldx, long long T, int C,
                                                            float* __restrict__ part) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), tl = threadIdx.x >> 5, b = blockIdx.z, B = gridDim.z;
  const float* xb = x + (long long)b * T * ldx;
  const bool ok = c < C;
  const float shift = ok ? xb[c] : 0.f;
  const long long t0 = blockIdx.y * INORM_PER, t1 = min(T, t0 + INORM_PER);
  float s1 = 0.f, s2 = 0.f;
  if (ok) instnorm_sums(xb, ldx, c, shift, t0, t1, tl, s1, s2);
  __shared__ float sh1[8][32], sh2[8][32];
  sh1[tl][threadIdx.x & 31] = s1; sh2[tl][threadIdx.x & 31] = s2;
  __syncthreads();
  if (tl != 0 || !ok) return;
  float a = 0.f, q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { a += sh1[i][threadIdx.x & 31]; q += sh2[i][threadIdx.x & 31]; }
  float* pp = part + ((long long)blockIdx.y * B + b) * 2 * C;
  pp[c] = a;
  pp[C + c] = q;
}

// y = norm(x) (+ GELU) element-wise from the summed statistics stats[b][{s1, s2}][c]
__global__ void instnorm_apply_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ stats,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int act_gelu,
                                      float* __restrict__ y, int ldy, int B, long long T, int C) {
  const long long total = (long long)B * T * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long p = i / C;
    const int b = (int)(p / T);
    const float* st = stats + (long long)b * 2 * C;
    const float shift = x[b * T * ldx + c];
    const float2 gb = instnorm_coef(st[c], st[C + c], (float)T, shift, gamma[c], beta[c], eps);
    y[p * ldy + c] = instnorm_apply(x[p * ldx + c], gb, act_gelu);
  }
}

}  // namespace evk
using namespace evk;
#define ST ((cudaStream_t)stream)

extern "C" int evk_layernorm_fwd(const float* x, int32_t ldx, const float* res, int32_t ldr, const float* gamma,
                                 const float* beta, float eps, float* y, int32_t ldy, float* stats, int64_t rows,
                                 int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && gamma && beta && y, EVK_ERR_ARG, "layernorm_fwd: null tensor");
  EVK_REQUIRE(C >= 1 && C <= 32 * LN_MAXV, EVK_ERR_UNSUPPORTED, "layernorm_fwd: C=%d unsupported", C);
  if (rows == 0) return EVK_OK;
  if (rows <= 8) {
    layernorm_fwd_block_kernel<<<(int)rows, 256, 0, ST>>>(x, ldx, res, ldr, gamma, beta, eps, y, ldy, stats, C);
    return check_launch("layernorm_fwd_block");
  }
  layernorm_fwd_kernel<<<cdiv(rows, 8), 256, 0, ST>>>(x, ldx, res, ldr, gamma, beta, eps, y, ldy, stats, rows, C);
  return check_launch("layernorm_fwd");
}

extern "C" int evk_layernorm_bwd(const float* x, int32_t ldx, const float* res, int32_t ldr, const float* gamma,
                                 const float* stats, const float* dy, int32_t lddy, float* dx, int32_t lddx,
                                 float* dgamma, float* dbeta, int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && gamma && stats && dy && dx && dgamma && dbeta, EVK_ERR_ARG, "layernorm_bwd: null tensor");
  EVK_REQUIRE(C >= 1 && C <= 32 * LN_MAXV, EVK_ERR_UNSUPPORTED, "layernorm_bwd: C=%d unsupported", C);
  if (rows == 0) return EVK_OK;
  int rpb = (int)((rows + kNumSMs * 4 - 1) / (kNumSMs * 4));
  if (rpb < 8) rpb = 8;
  const int S = cdiv(rows, rpb);
  Scratch part_buf((long long)S * 2 * C, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "layernorm_bwd: scratch allocation failed");
  layernorm_bwd_kernel<<<S, 256, 2 * C * sizeof(float), ST>>>(x, ldx, res, ldr, gamma, stats, dy, lddy, dx, lddx, part, nullptr, rows, C, rpb);
  if (int rc = check_launch("layernorm_bwd")) return rc;
  if (int rc = ordered_sum(part, S, 2ll * C, 1, 1, C, dgamma, 0, 0, ST)) return rc;
  return ordered_sum(part + C, S, 2ll * C, 1, 1, C, dbeta, 0, 0, ST);
}

extern "C" int evk_layernorm_drop_fwd(const float* x, const float* res, const float* gamma, const float* beta, float eps, float p,
                                      const uint64_t* rng, uint64_t sid, float* y, float* stats, int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && res && gamma && beta && y && stats && rng, EVK_ERR_ARG, "layernorm_drop_fwd: null tensor");
  EVK_REQUIRE(C >= 4 && (C % 4) == 0 && C <= 128 * LND_MAXV && p >= 0.f && p < 1.f, EVK_ERR_UNSUPPORTED, "layernorm_drop_fwd: C=%d p=%f unsupported", C, p);
  EVK_REQUIRE(((((uintptr_t)x) | ((uintptr_t)res) | ((uintptr_t)y)) & 15) == 0, EVK_ERR_ARG, "layernorm_drop_fwd: x / res / y must be 16-byte aligned");
  if (rows == 0) return EVK_OK;
  layernorm_drop_fwd_kernel<<<cdiv(rows, 8), 256, 0, ST>>>((const float4*)x, (const float4*)res, gamma, beta, eps, p,
                                                           (const unsigned long long*)rng, sid, (float4*)y, stats, rows, C / 4);
  return check_launch("layernorm_drop_fwd");
}

extern "C" int evk_layernorm_drop_bwd(const float* x, const float* res, const float* gamma, const float* stats, const float* dy, float p,
                                      const uint64_t* rng, uint64_t sid, float* dx, float* dres, float* dgamma, float* dbeta, int64_t rows,
                                      int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && res && gamma && stats && dy && dx && dres && dgamma && dbeta && rng, EVK_ERR_ARG, "layernorm_drop_bwd: null tensor");
  EVK_REQUIRE(C >= 4 && (C % 4) == 0 && C <= 128 * LND_MAXV, EVK_ERR_UNSUPPORTED, "layernorm_drop_bwd: C=%d unsupported", C);
  EVK_REQUIRE(((((uintptr_t)x) | ((uintptr_t)res) | ((uintptr_t)dy) | ((uintptr_t)dx) | ((uintptr_t)dres)) & 15) == 0, EVK_ERR_ARG,
              "layernorm_drop_bwd: x / res / dy / dx / dres must be 16-byte aligned");
  if (rows == 0) return EVK_OK;
  int rpb = (int)((rows + kNumSMs * 4 - 1) / (kNumSMs * 4));
  if (rpb < 8) rpb = 8;
  const int S = cdiv(rows, rpb);
  Scratch part_buf((long long)S * 2 * C, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "layernorm_drop_bwd: scratch allocation failed");
  layernorm_drop_bwd_kernel<<<S, 256, 2 * C * sizeof(float), ST>>>((const float4*)x, (const float4*)res, gamma, stats, (const float4*)dy, p,
                                                                   (const unsigned long long*)rng, sid, (float4*)dx, (float4*)dres, part, nullptr,
                                                                   rows, C / 4, rpb);
  if (int rc = check_launch("layernorm_drop_bwd")) return rc;
  if (int rc = ordered_sum(part, S, 2ll * C, 1, 1, C, dgamma, 0, 0, ST)) return rc;
  return ordered_sum(part + C, S, 2ll * C, 1, 1, C, dbeta, 0, 0, ST);
}

extern "C" int evk_colsum(const float* x, int64_t rows, int32_t n, int32_t ld, float* out, int32_t accumulate,
                          evk_stream_t stream) {
  EVK_REQUIRE(x && out && n >= 1, EVK_ERR_ARG, "colsum: bad arguments");
  if (!accumulate) {
    zero_kernel<<<cdiv(n, 256), 256, 0, ST>>>(out, n);
    int rc = check_launch("colsum_zero");
    if (rc) return rc;
  }
  if (rows == 0) return EVK_OK;
  int nb = cdiv(n, 32);
  long long want = ((long long)kNumSMs * 8 + nb - 1) / nb;
  int rpb = (int)((rows + want - 1) / want);
  if (rpb < 64) rpb = 64;
  dim3 grid(nb, cdiv(rows, rpb)), block(32, 8);
  EVK_REQUIRE(grid.y <= 65535, EVK_ERR_ARG, "colsum: grid too large");
  Scratch part_buf((long long)grid.y * n, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "colsum: scratch allocation failed");
  colsum_kernel<<<grid, block, 0, ST>>>(x, rows, n, ld, part, rpb);
  if (int rc = check_launch("colsum")) return rc;
  return ordered_sum(part, grid.y, 1, 1, n, out, 0, 0, ST);
}

extern "C" int evk_instnorm_cl(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, int32_t act_gelu, float* y,
                               int32_t ldy, int32_t B, int32_t T, int32_t C, const int32_t* lens, evk_stream_t stream) {
  EVK_REQUIRE(x && gamma && beta && y && B >= 1 && T >= 1 && C >= 1 && ldx >= C && ldy >= C, EVK_ERR_ARG, "instnorm_cl: bad arguments");
  instnorm_cl_kernel<<<dim3(cdiv(C, 32), B), 256, 0, ST>>>(x, ldx, gamma, beta, eps, act_gelu, y, ldy, T, C, lens);
  return check_launch("instnorm_cl");
}

extern "C" int evk_instnorm_plane(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, int32_t act_gelu,
                                  float* y, int32_t ldy, int32_t B, int64_t T, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && gamma && beta && y && B >= 1 && T >= 1 && C >= 1 && ldx >= C && ldy >= C, EVK_ERR_ARG,
              "instnorm_plane: bad arguments");
  const long long chunks = (T + INORM_PER - 1) / INORM_PER;
  EVK_REQUIRE(chunks <= 65535 && B <= 65535, EVK_ERR_ARG, "instnorm_plane: plane of %lld pixels too large", (long long)T);
  Scratch part_buf(chunks * B * 2 * C + (long long)B * 2 * C, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "instnorm_plane: scratch allocation failed");
  float* stats = part + chunks * B * 2 * C;
  instnorm_part_kernel<<<dim3(cdiv(C, 32), (unsigned)chunks, B), 256, 0, ST>>>(x, ldx, T, C, part);
  if (int rc = check_launch("instnorm_part")) return rc;
  zero_kernel<<<cdiv(2ll * B * C, 256), 256, 0, ST>>>(stats, 2 * B * C);
  if (int rc = check_launch("instnorm_zero")) return rc;
  if (int rc = ordered_sum(part, (int)chunks, (long long)B * 2 * C, 1, 1, B * 2 * C, stats, 0, 0, ST)) return rc;
  const long long total = (long long)B * T * C, blocks = (total + 255) / 256;
  instnorm_apply_kernel<<<(unsigned)(blocks < kNumSMs * 32 ? blocks : kNumSMs * 32), 256, 0, ST>>>(x, ldx, stats, gamma, beta, eps,
                                                                                                    act_gelu, y, ldy, B, T, C);
  return check_launch("instnorm_apply");
}
