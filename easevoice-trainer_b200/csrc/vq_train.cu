// The trainable semantic quantizer (freeze_quantizer: false): k-means initialisation, the EMA codebook update and the
// straight-through / commitment-loss pass.  Reference: core_vq.py:71-93 (kmeans), 141-149 (init_embed_), 203-228
// (EuclideanCodebook.forward), 301-318 (VectorQuantization.forward); models.py:917-927.
//
// Rows are the reference collate's shape: row (b, t) of a [B, T2, D] tensor takes part only when t < rows_ref[0] (a device
// scalar, T_ref / 2).  Every reduction runs in a fixed order and without float atomics, so the step is bit-reproducible.
#include "evk_common.cuh"

namespace evk {

constexpr int kMaxKmeansSamples = 500;     // core_vq.py:73

// samples[i] = the i-th valid row in (batch, frame) order, i < n = min(500, B * rows_ref); means[k] = samples[idx[k]] with
// idx drawn uniformly from [0, n) (sample_vectors with n < K: torch.randint) or injected
__global__ void kmeans_draw_kernel(const float* __restrict__ x, int ldx, int B, int T2, const int* __restrict__ rows_ref, int K,
                                   int D, const long long* __restrict__ idx_in, const unsigned long long* __restrict__ so,
                                   unsigned long long sid, float* __restrict__ samples, int* __restrict__ nsamp,
                                   float* __restrict__ means, long long* __restrict__ idx_out) {
  const int tr = min(rows_ref[0], T2);
  const int n = min(kMaxKmeansSamples, B * tr);
  if (blockIdx.x == 0 && threadIdx.x == 0) nsamp[0] = n;
  // blocks [0, 500): gather samples; blocks [500, 500 + K): pick the initial means
  if (blockIdx.x < kMaxKmeansSamples) {
    const int i = blockIdx.x;
    if (i >= n) return;
    const long long r = (long long)(i / tr) * T2 + i % tr;
    for (int d = threadIdx.x; d < D; d += blockDim.x) samples[(long long)i * D + d] = x[r * ldx + d];
    return;
  }
  const int k = blockIdx.x - kMaxKmeansSamples;
  if (k >= K || n == 0) return;
  long long j;
  if (idx_in) {
    j = idx_in[k];
  } else {
    const Philox rng(so[0]);
    const uint4 u = rng(so[1] + (unsigned long long)k, sid);
    j = (long long)(((unsigned long long)u.x | ((unsigned long long)u.y << 32)) % (unsigned long long)n);
  }
  if (threadIdx.x == 0 && idx_out) idx_out[k] = j;
  const long long r = (j / tr) * T2 + j % tr;
  for (int d = threadIdx.x; d < D; d += blockDim.x) means[(long long)k * D + d] = x[r * ldx + d];
}

// buckets[i] = argmax_k -sum_d (s_id - m_kd)^2 in the direct-difference form of core_vq.py:79-82, lowest index on ties
// (torch.max over a dim returns the first maximal index).  One block per sample; the sample stays in shared memory.
__global__ void __launch_bounds__(256) kmeans_assign_kernel(const float* __restrict__ samples, const int* __restrict__ nsamp,
                                                            const float* __restrict__ means, int K, int D,
                                                            int* __restrict__ buckets) {
  extern __shared__ float s[];
  __shared__ float bv[8];
  __shared__ int bi[8];
  const int i = blockIdx.x;
  if (i >= nsamp[0]) return;
  for (int d = threadIdx.x; d < D; d += blockDim.x) s[d] = samples[(long long)i * D + d];
  __syncthreads();
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float* m = means + (long long)k * D;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) {
      const float t = s[d] - m[d];
      acc += t * t;
    }
    const float dist = -acc;
    if (dist > best) { best = dist; besti = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = besti; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
    buckets[i] = besti;
  }
}

// bins[k] = |{i : buckets[i] == k}|; means[k] = (sum of its samples in sample order) / bins[k], kept when bins[k] == 0
// (core_vq.py:83-91).  One block per cluster.
__global__ void kmeans_update_kernel(const float* __restrict__ samples, const int* __restrict__ nsamp,
                                     const int* __restrict__ buckets, int K, int D, float* __restrict__ means,
                                     float* __restrict__ bins) {
  const int k = blockIdx.x;
  const int n = nsamp[0];
  int cnt = 0;
  for (int i = 0; i < n; ++i) cnt += buckets[i] == k;
  if (threadIdx.x == 0) bins[k] = (float)cnt;
  if (cnt == 0) return;
  const float c = (float)cnt;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < n; ++i)
      if (buckets[i] == k) acc += samples[(long long)i * D + d];
    means[(long long)k * D + d] = acc / c;
  }
}

// EMA of one code (core_vq.py:218-220): its rows are found in row order (a stable counting sort done per code: each
// 256-row chunk is compacted with warp ballots), their sum is accumulated in that order, then
// cluster_size <- decay * cs + (1 - decay) * count, embed_avg <- decay * ea + (1 - decay) * sum.
__global__ void __launch_bounds__(256) vq_ema_kernel(const float* __restrict__ x, int ldx, const long long* __restrict__ codes,
                                                     int B, int T2, const int* __restrict__ rows_ref, int K, int D,
                                                     float decay, float* __restrict__ cluster_size,
                                                     float* __restrict__ embed_avg) {
  constexpr int kCols = 4;                     // D <= 256 * kCols
  __shared__ int list[256];
  __shared__ int wcnt[8];
  const int k = blockIdx.x;
  const int tr = min(rows_ref[0], T2);
  const long long n = (long long)B * tr;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float acc[kCols] = {};
  int count = 0;
  for (long long c0 = 0; c0 < n; c0 += 256) {
    const long long i = c0 + threadIdx.x;
    long long r = 0;
    bool hit = false;
    if (i < n) {
      r = (i / tr) * T2 + i % tr;
      hit = codes[r] == k;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcnt[w] = __popc(m);
    __syncthreads();
    int base = 0, tot = 0;
    for (int j = 0; j < 8; ++j) {
      base += j < w ? wcnt[j] : 0;
      tot += wcnt[j];
    }
    if (hit) list[base + __popc(m & ((1u << lane) - 1u))] = (int)r;       // B * T2 < 2^31 (checked by the entry point)
    __syncthreads();
    for (int j = 0; j < tot; ++j) {
      const float* xr = x + (long long)list[j] * ldx;
#pragma unroll
      for (int q = 0; q < kCols; ++q) {
        const int d = threadIdx.x + q * 256;
        if (d < D) acc[q] += xr[d];
      }
    }
    count += tot;
    __syncthreads();
  }
  const float a = 1.f - decay;
  if (threadIdx.x == 0) cluster_size[k] = cluster_size[k] * decay + a * (float)count;
#pragma unroll
  for (int q = 0; q < kCols; ++q) {
    const int d = threadIdx.x + q * 256;
    if (d < D) embed_avg[(long long)k * D + d] = embed_avg[(long long)k * D + d] * decay + a * acc[q];
  }
}

// embed <- embed_avg / ((cs + eps) / (sum(cs) + K eps) * sum(cs))   (laplace_smoothing, core_vq.py:221-226).  Every block
// forms sum(cs) with the same tree, so all codes see the same value.
__global__ void vq_normalize_kernel(const float* __restrict__ cluster_size, const float* __restrict__ embed_avg, int K, int D,
                                    float eps, float* __restrict__ embed) {
  __shared__ float red[33];
  float s = 0.f;
  for (int j = threadIdx.x; j < K; j += blockDim.x) s += cluster_size[j];
  s = block_sum(s, red);
  const int k = blockIdx.x;
  const float cs = (cluster_size[k] + eps) / (s + (float)K * eps) * s;
  for (int d = threadIdx.x; d < D; d += blockDim.x) embed[(long long)k * D + d] = embed_avg[(long long)k * D + d] / cs;
}

// Straight-through value and commitment loss (core_vq.py:309-316, models.py:924-927):
//   qst = x + (q - x);  y[b][2t] = y[b][2t+1] = qst (nearest x2);  partial sums of (qst - x)^2 over the reference rows
__global__ void vq_st_fwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ q, int ldq, int B, int T2,
                                 int D, const int* __restrict__ rows_ref, float* __restrict__ y, float* __restrict__ qst,
                                 float* __restrict__ part) {
  __shared__ float red[33];
  const int tr = min(rows_ref[0], T2);
  const long long n = (long long)B * T2 * D;
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D;
    const int d = (int)(i - r * D);
    const int t = (int)(r % T2);
    const long long b = r / T2;
    const float xv = x[r * ldx + d];
    const float v = xv + (q[r * ldq + d] - xv);
    qst[i] = v;
    const long long o = (b * 2 * T2 + 2 * t) * D + d;
    y[o] = v;
    y[o + D] = v;
    if (t < tr) {
      const float e = v - xv;
      acc += e * e;
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// loss = sum(part) / (B * rows_ref * D), partials added in block order
__global__ void vq_mean_kernel(const float* __restrict__ part, int S, int B, int T2, int D, const int* __restrict__ rows_ref,
                               float* __restrict__ loss) {
  __shared__ float red[33];
  float s = 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) s += part[j];
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const long long N = (long long)B * min(rows_ref[0], T2) * D;
    loss[0] = N > 0 ? s / (float)N : 0.f;
  }
}

// dx = dy[2t] + dy[2t+1] + g * 2 (x - qst) / N on the reference rows, 0 past them
__global__ void vq_st_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, int ldx,
                                 const float* __restrict__ qst, int B, int T2, int D, const int* __restrict__ rows_ref,
                                 const float* __restrict__ gloss, float* __restrict__ dx) {
  const int tr = min(rows_ref[0], T2);
  const long long N = (long long)B * tr * D;
  const float g = N > 0 ? gloss[0] * 2.f / (float)N : 0.f;
  const long long n = (long long)B * T2 * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D;
    const int d = (int)(i - r * D);
    const int t = (int)(r % T2);
    const long long b = r / T2;
    float v = 0.f;
    if (t < tr) {
      const long long o = (b * 2 * T2 + 2 * t) * D + d;
      v = dy[o] + dy[o + D] + g * (x[r * ldx + d] - qst[i]);
    }
    dx[i] = v;
  }
}

// column sums over 64-row chunks: part[s][c] = sum_{r in chunk s} x[r][c] (ordered_sum adds the chunks in order)
__global__ void col_sum_part_kernel(const float* __restrict__ x, long long rows, int C, float* __restrict__ part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long r0 = (long long)blockIdx.y * 64;
  const long long r1 = min(rows, r0 + 64);
  float acc = 0.f;
  for (long long r = r0; r < r1; ++r) acc += x[r * C + c];
  part[(long long)blockIdx.y * C + c] = acc;
}

static inline unsigned grid_rows(long long n) {
  long long g = (n + 255) / 256;
  if (g > (long long)kNumSMs * 8) g = (long long)kNumSMs * 8;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace evk
using namespace evk;
#define ST ((cudaStream_t)stream)

extern "C" int evk_vq_kmeans_draw(const float* x, int32_t ldx, int32_t B, int32_t T2, const int32_t* rows_ref, int32_t K,
                                  int32_t D, const int64_t* idx, const uint64_t* seed_offset, uint64_t stream_id,
                                  float* samples, int32_t* nsamp, float* means, int64_t* idx_out, evk_stream_t stream) {
  EVK_REQUIRE(x && rows_ref && samples && nsamp && means && (idx || seed_offset) && B >= 1 && T2 >= 1 && K >= 1 && D >= 1,
              EVK_ERR_ARG, "vq_kmeans_draw: bad arguments");
  kmeans_draw_kernel<<<kMaxKmeansSamples + K, 256, 0, ST>>>(x, ldx, B, T2, rows_ref, K, D, (const long long*)idx,
                                                            (const unsigned long long*)seed_offset, stream_id, samples, nsamp,
                                                            means, (long long*)idx_out);
  return check_launch("vq_kmeans_draw");
}

extern "C" int evk_vq_kmeans_iter(const float* samples, const int32_t* nsamp, float* means, int32_t K, int32_t D,
                                  int32_t* buckets, float* bins, evk_stream_t stream) {
  EVK_REQUIRE(samples && nsamp && means && buckets && bins && K >= 1 && D >= 1 && D * 4 <= 48 * 1024, EVK_ERR_ARG,
              "vq_kmeans_iter: bad arguments");
  kmeans_assign_kernel<<<kMaxKmeansSamples, 256, D * sizeof(float), ST>>>(samples, nsamp, means, K, D, buckets);
  if (int rc = check_launch("vq_kmeans_assign")) return rc;
  kmeans_update_kernel<<<K, 256, 0, ST>>>(samples, nsamp, buckets, K, D, means, bins);
  return check_launch("vq_kmeans_update");
}

extern "C" int evk_vq_ema(const float* x, int32_t ldx, const int64_t* codes, int32_t B, int32_t T2, const int32_t* rows_ref,
                          float* cluster_size, float* embed_avg, float* embed, int32_t K, int32_t D, float decay, float eps,
                          evk_stream_t stream) {
  EVK_REQUIRE(x && codes && rows_ref && cluster_size && embed_avg && embed && K >= 1 && D >= 1 && D <= 1024 &&
                  (long long)B * T2 < (1ll << 31),
              EVK_ERR_ARG, "vq_ema: bad arguments");
  vq_ema_kernel<<<K, 256, 0, ST>>>(x, ldx, (const long long*)codes, B, T2, rows_ref, K, D, decay, cluster_size, embed_avg);
  if (int rc = check_launch("vq_ema")) return rc;
  vq_normalize_kernel<<<K, 256, 0, ST>>>(cluster_size, embed_avg, K, D, eps, embed);
  return check_launch("vq_normalize");
}

extern "C" int evk_vq_st_fwd(const float* x, int32_t ldx, const float* q, int32_t ldq, int32_t B, int32_t T2, int32_t D,
                             const int32_t* rows_ref, float* y, float* qst, float* loss, evk_stream_t stream) {
  EVK_REQUIRE(x && q && rows_ref && y && qst && loss && B >= 1 && T2 >= 1 && D >= 1, EVK_ERR_ARG, "vq_st_fwd: bad arguments");
  const unsigned g = grid_rows((long long)B * T2 * D);
  Scratch part_buf(g, ST);
  EVK_REQUIRE(part_buf.p, EVK_ERR_CUDA, "vq_st_fwd: scratch allocation failed");
  vq_st_fwd_kernel<<<g, 256, 0, ST>>>(x, ldx, q, ldq, B, T2, D, rows_ref, y, qst, part_buf.p);
  if (int rc = check_launch("vq_st_fwd")) return rc;
  vq_mean_kernel<<<1, 1024, 0, ST>>>(part_buf.p, (int)g, B, T2, D, rows_ref, loss);
  return check_launch("vq_mean");
}

extern "C" int evk_vq_st_bwd(const float* dy, const float* x, int32_t ldx, const float* qst, int32_t B, int32_t T2, int32_t D,
                             const int32_t* rows_ref, const float* gloss, float* dx, evk_stream_t stream) {
  EVK_REQUIRE(dy && x && qst && rows_ref && gloss && dx && B >= 1 && T2 >= 1 && D >= 1, EVK_ERR_ARG,
              "vq_st_bwd: bad arguments");
  vq_st_bwd_kernel<<<grid_rows((long long)B * T2 * D), 256, 0, ST>>>(dy, x, ldx, qst, B, T2, D, rows_ref, gloss, dx);
  return check_launch("vq_st_bwd");
}

extern "C" int evk_col_sum(const float* x, int64_t rows, int32_t C, float* out, evk_stream_t stream) {
  EVK_REQUIRE(x && out && rows >= 1 && C >= 1 && (rows + 63) / 64 <= 65535, EVK_ERR_ARG, "col_sum: bad arguments");
  const int S = (int)((rows + 63) / 64);
  Scratch part_buf((long long)S * C, ST);
  EVK_REQUIRE(part_buf.p, EVK_ERR_CUDA, "col_sum: scratch allocation failed");
  col_sum_part_kernel<<<dim3(cdiv(C, 128), S), 128, 0, ST>>>(x, rows, C, part_buf.p);
  if (int rc = check_launch("col_sum")) return rc;
  if (cudaMemsetAsync(out, 0, sizeof(float) * C, ST) != cudaSuccess) return check_launch("col_sum memset");
  return ordered_sum(part_buf.p, S, 1, 1, C, out, 0, 0, ST);
}
