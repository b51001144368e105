// Element-wise / row-wise kernels over channels-last [rows][C] views with explicit row pitches.
// All of these are HBM/L2-bandwidth bound: one thread per element (C fastest => coalesced), grid-stride.
// Reference call sites are listed per entry point in include/evk.h.
#include "evk_common.cuh"

namespace evk {

static inline dim3 grid1d(long long n, int bs = 256) {
  long long g = (n + bs - 1) / bs;
  if (g > (long long)kNumSMs * 32) g = (long long)kNumSMs * 32;   // grid-stride, a few waves of the SMs
  if (g < 1) g = 1;
  return dim3((unsigned)g);
}

#define EW_LOOP(i, n) for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float softplusf_(float x) { return x > 20.f ? x : log1pf(expf(x)); }

__global__ void unary_kernel(int op, float alpha, const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy,
                             long long rows, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    float v = x[r * ldx + c], o;
    switch (op) {
      case 0: o = v * alpha; break;
      case 1: o = v > 0.f ? v : v * alpha; break;
      case 2: o = tanhf(v); break;
      case 3: o = v * tanhf(softplusf_(v)); break;
      case 6: o = 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); break;     // exact (erf) GELU: HuBERT feature extractor / FFN, forward only
      default: o = fmaxf(v, 0.f); break;
    }
    y[r * ldy + c] = o;
  }
}

__global__ void unary_bwd_kernel(int op, float alpha, const float* __restrict__ x, int ldx, const float* __restrict__ dy,
                                 int lddy, float* __restrict__ dx, int lddx, long long rows, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    float v = x[r * ldx + c], g = dy[r * lddy + c], d;
    switch (op) {
      case 0: d = alpha; break;
      case 1: d = v > 0.f ? 1.f : alpha; break;
      case 2: { float t = tanhf(v); d = 1.f - t * t; } break;
      case 3: {  // d/dx x*tanh(softplus(x)) = tanh(sp) + x * (1 - tanh(sp)^2) * sigmoid(x)
        float sp = softplusf_(v), t = tanhf(sp);
        d = t + v * (1.f - t * t) * sigmoidf_(v);
      } break;
      case 5: d = 1.f - v * v; break;              // tanh, derivative taken from the OUTPUT y = tanh(x)
      default: d = v > 0.f ? 1.f : 0.f; break;
    }
    dx[r * lddx + c] = g * d;
  }
}

__global__ void axpby_kernel(const float* __restrict__ a, int lda, float alpha, const float* __restrict__ b, int ldb,
                             float beta, const float* __restrict__ c3, int ldc, float gamma, float* __restrict__ y,
                             int ldy, long long rows, int C, const int* __restrict__ len, int T) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    float v = alpha * a[r * lda + c];
    if (b) v += beta * b[r * ldb + c];
    if (c3) v += gamma * c3[r * ldc + c];
    if (len) {
      long long bb = r / T;
      int t = (int)(r - bb * T);
      if (t >= len[bb]) v = 0.f;
    }
    y[r * ldy + c] = v;
  }
}

__global__ void add_bvec_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ v, int ldv,
                                float* __restrict__ y, int ldy, long long rows, int T, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    long long b = r / T;
    y[r * ldy + c] = x[r * ldx + c] + v[b * ldv + c];
  }
}

__global__ void wn_gate_kernel(const float* __restrict__ a, int lda, const float* __restrict__ g, int ldg,
                               float* __restrict__ o, int ldo, long long rows, int T, int H) {
  EW_LOOP(i, rows * H) {
    long long r = i / H;
    int c = (int)(i - r * H);
    long long b = r / T;
    float ta = a[r * lda + c], sa = a[r * lda + H + c];
    if (g) { ta += g[b * ldg + c]; sa += g[b * ldg + H + c]; }
    o[r * ldo + c] = tanhf(ta) * sigmoidf_(sa);
  }
}

__global__ void wn_gate_bwd_kernel(const float* __restrict__ a, int lda, const float* __restrict__ g, int ldg,
                                   const float* __restrict__ dact, int lddo, float* __restrict__ da, int ldda,
                                   long long rows, int T, int H) {
  EW_LOOP(i, rows * H) {
    long long r = i / H;
    int c = (int)(i - r * H);
    long long b = r / T;
    float ta = a[r * lda + c], sa = a[r * lda + H + c];
    if (g) { ta += g[b * ldg + c]; sa += g[b * ldg + H + c]; }
    float t = tanhf(ta), s = sigmoidf_(sa), d = dact[r * lddo + c];
    da[r * ldda + c] = d * s * (1.f - t * t);
    da[r * ldda + H + c] = d * t * s * (1.f - s);
  }
}

__global__ void glu_res_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ h, int ldh,
                               float* __restrict__ y, int ldy, long long rows, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    y[r * ldy + c] = (x ? x[r * ldx + c] : 0.f) + h[r * ldh + c] * sigmoidf_(h[r * ldh + C + c]);
  }
}

__global__ void glu_res_bwd_kernel(const float* __restrict__ h, int ldh, const float* __restrict__ dy, int lddy,
                                   float* __restrict__ dh, int lddh, long long rows, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    float h1 = h[r * ldh + c], s = sigmoidf_(h[r * ldh + C + c]), d = dy[r * lddy + c];
    dh[r * lddh + c] = d * s;
    dh[r * lddh + C + c] = d * h1 * s * (1.f - s);
  }
}

__global__ void reparam_kernel(const float* __restrict__ st, int lds, const float* __restrict__ nz, int ldn,
                               float* __restrict__ z, int ldz, long long rows, int T, int C,
                               const int* __restrict__ len) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    long long b = r / T;
    int t = (int)(r - b * T);
    float v = st[r * lds + c] + nz[r * ldn + c] * __expf(st[r * lds + C + c]);
    z[r * ldz + c] = (len && t >= len[b]) ? 0.f : v;
  }
}

__global__ void reparam_bwd_kernel(const float* __restrict__ st, int lds, const float* __restrict__ nz, int ldn,
                                   const float* __restrict__ dz, int lddz, float* __restrict__ ds, int ldds,
                                   long long rows, int T, int C, const int* __restrict__ len) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    long long b = r / T;
    int t = (int)(r - b * T);
    float g = (len && t >= len[b]) ? 0.f : dz[r * lddz + c];
    ds[r * ldds + c] = g;
    ds[r * ldds + C + c] = g * nz[r * ldn + c] * __expf(st[r * lds + C + c]);
  }
}

__global__ void rowmask_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, long long rows,
                               int T, int C, const int* __restrict__ len) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    long long b = r / T;
    int t = (int)(r - b * T);
    y[r * ldy + c] = (t < len[b]) ? x[r * ldx + c] : 0.f;
  }
}

__global__ void flip_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, long long rows, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    y[r * ldy + c] = x[r * ldx + (C - 1 - c)];
  }
}

__global__ void slice_rows_kernel(const float* __restrict__ x, int ldx, int Tin, const long long* __restrict__ ids,
                                  int mul, float* __restrict__ y, int ldy, int B, int seg, int C, int scatter) {
  EW_LOOP(i, (long long)B * seg * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    int b = (int)(r / seg), j = (int)(r - (long long)b * seg);
    long long src = (long long)b * Tin + ids[b] * mul + j;
    if (scatter) const_cast<float*>(x)[src * ldx + c] = y[r * ldy + c];
    else y[r * ldy + c] = x[src * ldx + c];
  }
}

__global__ void reflect_pad_right_kernel(const float* __restrict__ x, int T, float* __restrict__ y, int Tp, int B, int bwd) {
  if (!bwd) {
    EW_LOOP(i, (long long)B * Tp) {
      int b = (int)(i / Tp), t = (int)(i - (long long)b * Tp);
      int s = t < T ? t : 2 * (T - 1) - t;
      y[i] = x[(long long)b * T + s];
    }
  } else {  // x = dX [B][T] written, y = dY [B][Tp] read
    EW_LOOP(i, (long long)B * T) {
      int b = (int)(i / T), t = (int)(i - (long long)b * T);
      float v = y[(long long)b * Tp + t];
      int m = 2 * (T - 1) - t;                       // mirrored position in the padded tail
      if (m >= T && m < Tp) v += y[(long long)b * Tp + m];
      const_cast<float*>(x)[i] = v;
    }
  }
}

// tiled transpose [B][C][T] -> [B][T][ld] (to_btc) or back
__global__ void transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int T, int ld, int to_btc) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const float* xb;
  float* yb;
  if (to_btc) {
    xb = x + (long long)b * C * T; yb = y + (long long)b * T * ld;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      int c = c0 + i, t = t0 + threadIdx.x;
      tile[i][threadIdx.x] = (c < C && t < T) ? xb[(long long)c * T + t] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      int t = t0 + i, c = c0 + threadIdx.x;
      if (t < T && c < C) yb[(long long)t * ld + c] = tile[threadIdx.x][i];
    }
  } else {
    xb = x + (long long)b * T * ld; yb = y + (long long)b * C * T;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      int t = t0 + i, c = c0 + threadIdx.x;
      tile[i][threadIdx.x] = (c < C && t < T) ? xb[(long long)t * ld + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      int c = c0 + i, t = t0 + threadIdx.x;
      if (t < T && c < C) yb[(long long)c * T + t] = tile[threadIdx.x][i];
    }
  }
}

// [B][T][ldx] (C valid) -> [B][C][ldy] (T + shift valid): y[b][c][u] = x[b][u - shift][c], zero for u < shift.
// The contraction index of a weight gradient becomes contiguous.
__global__ void transpose_rows_kernel(const float* __restrict__ x, int ldx, long long x_sb, float* __restrict__ y, int ldy,
                                      long long y_sb, int T, int C, int shift) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const float* xb = x + b * x_sb;
  float* yb = y + b * y_sb;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int t = t0 + i - shift, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t >= 0 && t < T) ? xb[(long long)t * ldx + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, u = t0 + threadIdx.x;
    if (u < T + shift && c < C) yb[(long long)c * ldy + u] = tile[threadIdx.x][i];
  }
}

// all delayed copies of evk_transpose_rows in one pass over x: y[r][b][c][u] = x[b][u - r][c] for every r in `mask`
// (bit r set, r = 0..3); the 32 x 32 tile is loaded once with a 3-row halo.
__global__ void transpose_rows_multi_kernel(const float* __restrict__ x, int ldx, long long x_sb, float* __restrict__ y, int ldy,
                                            long long y_sb, long long y_rs, int T, int C, int mask) {
  __shared__ float tile[35][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const float* xb = x + b * x_sb;
  for (int i = threadIdx.y; i < 35; i += blockDim.y) {
    int t = t0 + i - 3, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t >= 0 && t < T) ? xb[(long long)t * ldx + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if (!((mask >> r) & 1)) continue;
    float* yb = y + r * y_rs + b * y_sb;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      int c = c0 + i, u = t0 + threadIdx.x;
      if (u < T + r && c < C) yb[(long long)c * ldy + u] = tile[threadIdx.x + 3 - r][i];
    }
  }
}

// One pass over an output gradient for everything a conv's backward needs from it (round 1 ran three kernels -- activation
// backward, transpose for the TMA weight gradient, column sums for the bias -- and four trips through memory):
//   g[t][c]    = dy[t][c] * act'(y[t][c]) * (t < len*P)        -> dpre  (normal layout, only when it differs from dy)
//   dyt[c][t]  = g[t][c]                                        -> the K-major A operand of the weight-gradient GEMM
//   dbias[c]  += sum_t g[t][c]                                  (one partial per column per block, summed in block order)
constexpr int DYP_ROWS = 128;          // rows per block: 16 independent loads per thread in flight, one barrier
__global__ void __launch_bounds__(256) dy_prep_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ yact, int ldy, int act,
                                                      float slope, float gscale, const int* __restrict__ len, int P, float* __restrict__ dpre,
                                                      int ldp, float* __restrict__ dyt, int ldt, long long t_sb, float* __restrict__ dbias, int T,
                                                      int C) {
  __shared__ float tile[DYP_ROWS][33];
  __shared__ float csum[8][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * DYP_ROWS, tx = threadIdx.x, ty = threadIdx.y;
  const long long row0 = (long long)b * T;
  const int lim = len ? len[b] * P : 0x7fffffff;
  const int c = c0 + tx;
  float v[DYP_ROWS / 8], o[DYP_ROWS / 8];
#pragma unroll
  for (int k = 0; k < DYP_ROWS / 8; ++k) {                       // all loads first (memory-level parallelism)
    const int t = t0 + ty + 8 * k;
    const bool in = c < C && t < T;
    v[k] = in ? dy[(row0 + t) * lddy + c] : 0.f;
    o[k] = (in && act) ? yact[(row0 + t) * ldy + c] : 1.f;
  }
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < DYP_ROWS / 8; ++k) {
    const int t = t0 + ty + 8 * k;
    float g = v[k] * gscale;
    if (act) g *= (act == EVK_ACT_LRELU) ? (o[k] > 0.f ? 1.f : slope) : (act == EVK_ACT_RELU) ? (o[k] > 0.f ? 1.f : 0.f) : (1.f - o[k] * o[k]);
    if (t >= lim) g = 0.f;
    if (dpre && c < C && t < T) dpre[(row0 + t) * ldp + c] = g;
    tile[ty + 8 * k][tx] = g;
    acc += g;
  }
  __syncthreads();
  if (dyt) {
#pragma unroll
    for (int i = ty; i < 32; i += 8) {
      const int cc = c0 + i;
      if (cc < C) {
        float* dst = dyt + b * t_sb + (long long)cc * ldt + t0;
#pragma unroll
        for (int k = 0; k < DYP_ROWS / 32; ++k) {
          const int u = tx + 32 * k;
          if (t0 + u < T) dst[u] = tile[u][i];
        }
      }
    }
  }
  if (dbias) {
    csum[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && c < C) {
      float sacc = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) sacc += csum[k][tx];
      dbias[((long long)blockIdx.z * gridDim.x + blockIdx.x) * C + c] = sacc;    // partial of this block (ordered_sum)
    }
  }
}

// stride-phase split: xs[rho][b][j*P + w][c] = x[b][(j*s + rho)*P + w][c] (zero when j*s + rho >= T), j < Jp
__global__ void phase_split_kernel(const float* __restrict__ x, int ldx, long long x_sb, float* __restrict__ xs, long long xs_ps,
                                   int B, int T, int P, int C, int s, int Jp) {
  const int c4n = C / 4;
  const long long n = (long long)s * B * Jp * P * c4n;
  EW_LOOP(i, n) {
    int c4 = (int)(i % c4n);
    long long r = i / c4n;
    int w = (int)(r % P); r /= P;
    int j = (int)(r % Jp); r /= Jp;
    int b = (int)(r % B);
    int rho = (int)(r / B);
    const int t = j * s + rho;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < T) v = *reinterpret_cast<const float4*>(x + b * x_sb + ((long long)t * P + w) * ldx + c4 * 4);
    *reinterpret_cast<float4*>(xs + rho * xs_ps + (((long long)b * Jp + j) * P + w) * C + c4 * 4) = v;
  }
}

__global__ void embedding_kernel(const float* __restrict__ tab, int ldt, const long long* __restrict__ idx, long long rows,
                                 int rep, float* __restrict__ y, int ldy, int C) {
  EW_LOOP(i, rows * C) {
    long long r = i / C;
    int c = (int)(i - r * C);
    y[r * ldy + c] = tab[idx[r / rep] * ldt + c];
  }
}

// dtab[idx[r]][c] += dy[r][c] without atomics, in two passes: thread (chunk, c) adds the rows of its EMB_CHUNK-row chunk in
// row order into part[chunk][idx][c] (zeroed first), then ordered_sum adds the chunks in order.
constexpr int EMB_CHUNK = 256;
__global__ void embedding_bwd_kernel(const float* __restrict__ dy, int lddy, const long long* __restrict__ idx,
                                     long long rows, float* __restrict__ part, int V, int C) {
  const long long nchunks = (rows + EMB_CHUNK - 1) / EMB_CHUNK;
  EW_LOOP(i, nchunks * C) {
    const int c = (int)(i % C);
    const long long k = i / C;
    float* pk = part + k * V * (long long)C + c;
    const long long r1 = min(rows, (k + 1) * EMB_CHUNK);
    for (long long r = k * EMB_CHUNK; r < r1; ++r) pk[idx[r] * C] += dy[r * lddy + c];
  }
}

// one block per (b, channel-chunk of 32): masked mean over time
__global__ void masked_mean_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, int T, int C,
                                   const int* __restrict__ len, int bwd) {
  const int b = blockIdx.y, c = blockIdx.x * 32 + (threadIdx.x & 31), ty = threadIdx.x >> 5, ny = blockDim.x >> 5;
  const int n = len ? min(len[b], T) : T;
  if (!bwd) {
    __shared__ float part[8][33];
    float acc = 0.f;
    if (c < C)
      for (int t = ty; t < n; t += ny) acc += x[((long long)b * T + t) * ldx + c];
    part[ty][threadIdx.x & 31] = acc;
    __syncthreads();
    if (ty == 0 && c < C) {
      float s = 0.f;
      for (int k = 0; k < ny; ++k) s += part[k][threadIdx.x];
      y[(long long)b * ldy + c] = s / (float)n;
    }
  } else {  // x is dX (written) [B][T][C], y is dY [B][C]
    if (c < C) {
      const float g = y[(long long)b * ldy + c] / (float)n;
      for (int t = ty; t < T; t += ny) const_cast<float*>(x)[((long long)b * T + t) * ldx + c] = t < n ? g : 0.f;
    }
  }
}

__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float p,
                               const unsigned long long* __restrict__ so, unsigned long long sid) {
  const Philox rng(so[0]);
  const unsigned long long base = so[1];
  const float scale = 1.f / (1.f - p);
  const long long n4 = (n + 3) / 4;
  EW_LOOP(i, n4) {
    uint4 r = rng(base + (unsigned long long)i, sid);
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      long long e = i * 4 + k;
      if (e < n) y[e] = (u32_to_unit(rr[k]) >= p) ? x[e] * scale : 0.f;
    }
  }
}

__global__ void randn_kernel(float* __restrict__ y, long long n, const unsigned long long* __restrict__ so,
                             unsigned long long sid) {
  const Philox rng(so[0]);
  const unsigned long long base = so[1];
  const long long n4 = (n + 3) / 4;
  EW_LOOP(i, n4) {
    uint4 r = rng(base + (unsigned long long)i, sid);
    // Box-Muller on two pairs
    float u1 = fmaxf(u32_to_unit(r.x), 5.9604645e-8f), u2 = u32_to_unit(r.y);
    float u3 = fmaxf(u32_to_unit(r.z), 5.9604645e-8f), u4 = u32_to_unit(r.w);
    float m1 = sqrtf(-2.f * logf(u1)), m2 = sqrtf(-2.f * logf(u3));
    float s1, c1, s2, c2;
    sincosf(6.283185307179586f * u2, &s1, &c1);
    sincosf(6.283185307179586f * u4, &s2, &c2);
    const float o[4] = {m1 * c1, m1 * s1, m2 * c2, m2 * s2};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      long long e = i * 4 + k;
      if (e < n) y[e] = o[k];
    }
  }
}

__global__ void rand_slice_ids_kernel(long long* __restrict__ ids, const int* __restrict__ len, int B, int seg,
                                      const unsigned long long* __restrict__ so, unsigned long long sid) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const Philox rng(so[0]);
  uint4 r = rng(so[1] + (unsigned long long)b, sid);
  const int mx = len[b] - seg + 1;                   // commons.py:55-56: (rand * ids_str_max).long()
  long long v = (long long)(u32_to_unit(r.x) * (float)mx);
  if (v > mx - 1) v = mx - 1;
  if (v < 0) v = 0;
  ids[b] = v;
}

__global__ void advance_rng_kernel(unsigned long long* so, unsigned long long inc) { so[1] += inc; }

}  // namespace evk
using namespace evk;

#define ST ((cudaStream_t)stream)

extern "C" int evk_unary(int32_t op, float alpha, const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows,
                         int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && y && ((op >= 0 && op <= 4) || op == 6), EVK_ERR_ARG, "unary: bad arguments");
  if (rows * C == 0) return EVK_OK;
  unary_kernel<<<grid1d(rows * C), 256, 0, ST>>>(op, alpha, x, ldx, y, ldy, rows, C);
  return check_launch("unary");
}
extern "C" int evk_unary_bwd(int32_t op, float alpha, const float* x, int32_t ldx, const float* dy, int32_t lddy,
                             float* dx, int32_t lddx, int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && dy && dx && op >= 0 && op <= 5, EVK_ERR_ARG, "unary_bwd: bad arguments");
  if (rows * C == 0) return EVK_OK;
  unary_bwd_kernel<<<grid1d(rows * C), 256, 0, ST>>>(op, alpha, x, ldx, dy, lddy, dx, lddx, rows, C);
  return check_launch("unary_bwd");
}
extern "C" int evk_axpby(const float* a, int32_t lda, float alpha, const float* b, int32_t ldb, float beta,
                         const float* c, int32_t ldc, float gamma, float* y, int32_t ldy, int64_t rows, int32_t C,
                         const int32_t* len, int32_t T, evk_stream_t stream) {
  EVK_REQUIRE(a && y && (!len || T > 0), EVK_ERR_ARG, "axpby: bad arguments");
  if (rows * C == 0) return EVK_OK;
  axpby_kernel<<<grid1d(rows * C), 256, 0, ST>>>(a, lda, alpha, b, ldb, beta, c, ldc, gamma, y, ldy, rows, C, len, T);
  return check_launch("axpby");
}
extern "C" int evk_add_bvec(const float* x, int32_t ldx, const float* v, int32_t ldv, float* y, int32_t ldy, int32_t B,
                            int32_t T, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && v && y, EVK_ERR_ARG, "add_bvec: null tensor");
  long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  add_bvec_kernel<<<grid1d(rows * C), 256, 0, ST>>>(x, ldx, v, ldv, y, ldy, rows, T, C);
  return check_launch("add_bvec");
}
extern "C" int evk_wn_gate(const float* a, int32_t lda, const float* g, int32_t ldg, float* acts, int32_t ldo, int32_t B,
                           int32_t T, int32_t Hc, evk_stream_t stream) {
  EVK_REQUIRE(a && acts, EVK_ERR_ARG, "wn_gate: null tensor");
  long long rows = (long long)B * T;
  if (rows * Hc == 0) return EVK_OK;
  wn_gate_kernel<<<grid1d(rows * Hc), 256, 0, ST>>>(a, lda, g, ldg, acts, ldo, rows, T, Hc);
  return check_launch("wn_gate");
}
extern "C" int evk_wn_gate_bwd(const float* a, int32_t lda, const float* g, int32_t ldg, const float* dacts,
                               int32_t lddo, float* da, int32_t ldda, int32_t B, int32_t T, int32_t Hc,
                               evk_stream_t stream) {
  EVK_REQUIRE(a && dacts && da, EVK_ERR_ARG, "wn_gate_bwd: null tensor");
  long long rows = (long long)B * T;
  if (rows * Hc == 0) return EVK_OK;
  wn_gate_bwd_kernel<<<grid1d(rows * Hc), 256, 0, ST>>>(a, lda, g, ldg, dacts, lddo, da, ldda, rows, T, Hc);
  return check_launch("wn_gate_bwd");
}
extern "C" int evk_glu_res(const float* x, int32_t ldx, const float* h, int32_t ldh, float* y, int32_t ldy,
                           int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(h && y, EVK_ERR_ARG, "glu_res: null tensor");
  if (rows * C == 0) return EVK_OK;
  glu_res_kernel<<<grid1d(rows * C), 256, 0, ST>>>(x, ldx, h, ldh, y, ldy, rows, C);
  return check_launch("glu_res");
}
extern "C" int evk_glu_res_bwd(const float* h, int32_t ldh, const float* dy, int32_t lddy, float* dh, int32_t lddh,
                               int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(h && dy && dh, EVK_ERR_ARG, "glu_res_bwd: null tensor");
  if (rows * C == 0) return EVK_OK;
  glu_res_bwd_kernel<<<grid1d(rows * C), 256, 0, ST>>>(h, ldh, dy, lddy, dh, lddh, rows, C);
  return check_launch("glu_res_bwd");
}
extern "C" int evk_reparam(const float* stats, int32_t lds, const float* noise, int32_t ldn, float* z, int32_t ldz,
                           int32_t B, int32_t T, int32_t C, const int32_t* len, evk_stream_t stream) {
  EVK_REQUIRE(stats && noise && z, EVK_ERR_ARG, "reparam: null tensor");
  long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  reparam_kernel<<<grid1d(rows * C), 256, 0, ST>>>(stats, lds, noise, ldn, z, ldz, rows, T, C, len);
  return check_launch("reparam");
}
extern "C" int evk_reparam_bwd(const float* stats, int32_t lds, const float* noise, int32_t ldn, const float* dz,
                               int32_t lddz, float* dstats, int32_t ldds, int32_t B, int32_t T, int32_t C,
                               const int32_t* len, evk_stream_t stream) {
  EVK_REQUIRE(stats && noise && dz && dstats, EVK_ERR_ARG, "reparam_bwd: null tensor");
  long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  reparam_bwd_kernel<<<grid1d(rows * C), 256, 0, ST>>>(stats, lds, noise, ldn, dz, lddz, dstats, ldds, rows, T, C, len);
  return check_launch("reparam_bwd");
}
extern "C" int evk_rowmask(const float* x, int32_t ldx, float* y, int32_t ldy, int32_t B, int32_t T, int32_t C,
                           const int32_t* len, evk_stream_t stream) {
  EVK_REQUIRE(x && y && len, EVK_ERR_ARG, "rowmask: null tensor");
  long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  rowmask_kernel<<<grid1d(rows * C), 256, 0, ST>>>(x, ldx, y, ldy, rows, T, C, len);
  return check_launch("rowmask");
}
extern "C" int evk_flip_channels(const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows, int32_t C,
                                 evk_stream_t stream) {
  EVK_REQUIRE(x && y && x != y, EVK_ERR_ARG, "flip_channels: bad arguments");
  if (rows * C == 0) return EVK_OK;
  flip_kernel<<<grid1d(rows * C), 256, 0, ST>>>(x, ldx, y, ldy, rows, C);
  return check_launch("flip_channels");
}
extern "C" int evk_slice_rows(const float* x, int32_t ldx, int32_t Tin, const int64_t* ids, int32_t mul, float* y,
                              int32_t ldy, int32_t B, int32_t seg, int32_t C, int32_t scatter, evk_stream_t stream) {
  EVK_REQUIRE(x && y && ids, EVK_ERR_ARG, "slice_rows: null tensor");
  long long n = (long long)B * seg * C;
  if (n == 0) return EVK_OK;
  slice_rows_kernel<<<grid1d(n), 256, 0, ST>>>(x, ldx, Tin, (const long long*)ids, mul, y, ldy, B, seg, C, scatter);
  return check_launch("slice_rows");
}
extern "C" int evk_reflect_pad_right(const float* x, int32_t T, float* y, int32_t Tp, int32_t B, int32_t bwd,
                                     evk_stream_t stream) {
  EVK_REQUIRE(x && y && Tp >= T && Tp - T < T, EVK_ERR_ARG, "reflect_pad_right: bad arguments");
  long long n = (long long)B * (bwd ? T : Tp);
  if (n == 0) return EVK_OK;
  reflect_pad_right_kernel<<<grid1d(n), 256, 0, ST>>>(x, T, y, Tp, B, bwd);
  return check_launch("reflect_pad_right");
}
extern "C" int evk_transpose_bct_btc(const float* x, float* y, int32_t B, int32_t C, int32_t T, int32_t ld,
                                     int32_t to_btc, evk_stream_t stream) {
  EVK_REQUIRE(x && y && ld >= C, EVK_ERR_ARG, "transpose: bad arguments");
  if ((long long)B * C * T == 0) return EVK_OK;
  dim3 grid(cdiv(T, 32), cdiv(C, 32), B), block(32, 8);
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "transpose: grid too large");
  transpose_kernel<<<grid, block, 0, ST>>>(x, y, C, T, ld, to_btc);
  return check_launch("transpose");
}
extern "C" int evk_transpose_rows(const float* x, int32_t ldx, int64_t x_sb, float* y, int32_t ldy, int64_t y_sb, int32_t B, int32_t T,
                                  int32_t C, int32_t shift, evk_stream_t stream) {
  EVK_REQUIRE(x && y && ldx >= C && shift >= 0 && ldy >= T + shift, EVK_ERR_ARG, "transpose_rows: bad arguments");
  if ((long long)B * C * T == 0) return EVK_OK;
  dim3 grid(cdiv(T + shift, 32), cdiv(C, 32), B), block(32, 8);
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "transpose_rows: grid too large");
  transpose_rows_kernel<<<grid, block, 0, ST>>>(x, ldx, x_sb, y, ldy, y_sb, T, C, shift);
  return check_launch("transpose_rows");
}
extern "C" int evk_transpose_rows_multi(const float* x, int32_t ldx, int64_t x_sb, float* y, int32_t ldy, int64_t y_sb, int64_t y_rs,
                                        int32_t B, int32_t T, int32_t C, int32_t mask, evk_stream_t stream) {
  EVK_REQUIRE(x && y && ldx >= C && ldy >= T + 3 && mask > 0 && mask < 16, EVK_ERR_ARG, "transpose_rows_multi: bad arguments");
  if ((long long)B * C * T == 0) return EVK_OK;
  dim3 grid(cdiv(T + 3, 32), cdiv(C, 32), B), block(32, 8);
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "transpose_rows_multi: grid too large");
  transpose_rows_multi_kernel<<<grid, block, 0, ST>>>(x, ldx, x_sb, y, ldy, y_sb, y_rs, T, C, mask);
  return check_launch("transpose_rows_multi");
}
// dy [B][T][lddy] (T rows per batch item), yact = the conv's activated OUTPUT (nullable when act == 0), len (nullable int32 [B],
// rows t >= len[b] * P are zeroed), outputs each nullable: dpre [B][T][ldp], dyt [B][C][ldt] (batch pitch t_sb), dbias [C]
// (accumulated: zero it first).
extern "C" int evk_dy_prep(const float* dy, int32_t lddy, const float* yact, int32_t ldy, int32_t act, float slope, float gscale,
                           const int32_t* len, int32_t P, float* dpre, int32_t ldp, float* dyt, int32_t ldt, int64_t t_sb, float* dbias,
                           int32_t B, int32_t T, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(dy && (act == 0 || yact) && act >= 0 && act <= 3 && P >= 1 && (dpre || dyt || dbias), EVK_ERR_ARG, "dy_prep: bad arguments");
  EVK_REQUIRE(!dyt || ldt >= T, EVK_ERR_ARG, "dy_prep: ldt too small");
  if ((long long)B * T * C == 0) return EVK_OK;
  dim3 grid(cdiv(T, DYP_ROWS), cdiv(C, 32), B), block(32, 8);
  EVK_REQUIRE(grid.y <= 65535 && grid.z <= 65535, EVK_ERR_ARG, "dy_prep: grid too large");
  const int S = (int)(grid.x * grid.z);
  Scratch part_buf(dbias ? (long long)S * C : 0, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(!dbias || part, EVK_ERR_CUDA, "dy_prep: scratch allocation failed");
  dy_prep_kernel<<<grid, block, 0, ST>>>(dy, lddy, yact, ldy, act, slope, gscale, len, P, dpre, ldp, dyt, ldt, t_sb, part, T, C);
  if (int rc = check_launch("dy_prep")) return rc;
  return dbias ? ordered_sum(part, S, 1, 1, C, dbias, 0, 0, ST) : EVK_OK;
}
extern "C" int evk_phase_split(const float* x, int32_t ldx, int64_t x_sb, float* xs, int64_t xs_ps, int32_t B, int32_t T, int32_t P,
                               int32_t C, int32_t stride, int32_t Jp, evk_stream_t stream) {
  EVK_REQUIRE(x && xs && (C % 4) == 0 && (ldx % 4) == 0 && (x_sb % 4) == 0 && (xs_ps % 4) == 0 && stride >= 1 && Jp * stride >= T,
              EVK_ERR_ARG, "phase_split: bad arguments");
  long long n = (long long)stride * B * Jp * P * (C / 4);
  if (n == 0) return EVK_OK;
  phase_split_kernel<<<grid1d(n), 256, 0, ST>>>(x, ldx, x_sb, xs, xs_ps, B, T, P, C, stride, Jp);
  return check_launch("phase_split");
}
extern "C" int evk_embedding(const float* table, int32_t ldt, const int64_t* idx, int64_t rows, int32_t rep, float* y,
                             int32_t ldy, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(rep >= 1, EVK_ERR_ARG, "embedding: bad arguments");
  if (rows * C == 0) return EVK_OK;                          // nothing to read or write (an empty tensor may have a null pointer)
  EVK_REQUIRE(table && idx && y, EVK_ERR_ARG, "embedding: bad arguments");
  embedding_kernel<<<grid1d(rows * C), 256, 0, ST>>>(table, ldt, (const long long*)idx, rows, rep, y, ldy, C);
  return check_launch("embedding");
}
extern "C" int evk_embedding_bwd(const float* dy, int32_t lddy, const int64_t* idx, int64_t rows, float* dtable,
                                 int32_t ldt, int32_t C, int32_t V, evk_stream_t stream) {
  EVK_REQUIRE(dy && idx && dtable && V > 0, EVK_ERR_ARG, "embedding_bwd: null tensor or empty table");
  if (rows * C == 0) return EVK_OK;
  const long long nchunks = (rows + EMB_CHUNK - 1) / EMB_CHUNK;
  Scratch part_buf(nchunks * V * (long long)C, ST);
  EVK_REQUIRE(part_buf.p, EVK_ERR_CUDA, "embedding_bwd: scratch allocation failed");
  if (cudaMemsetAsync(part_buf.p, 0, (size_t)nchunks * V * C * sizeof(float), ST) != cudaSuccess) return check_launch("embedding_bwd_zero");
  embedding_bwd_kernel<<<grid1d(nchunks * C), 256, 0, ST>>>(dy, lddy, (const long long*)idx, rows, part_buf.p, V, C);
  if (int rc = check_launch("embedding_bwd")) return rc;
  return ordered_sum(part_buf.p, (int)nchunks, 1, V, C, dtable, 0, ldt, ST);
}
extern "C" int evk_masked_mean(const float* x, int32_t ldx, float* y, int32_t ldy, int32_t B, int32_t T, int32_t C,
                               const int32_t* len, int32_t bwd, evk_stream_t stream) {
  EVK_REQUIRE(x && y, EVK_ERR_ARG, "masked_mean: null tensor");
  if ((long long)B * T * C == 0) return EVK_OK;
  dim3 grid(cdiv(C, 32), B);
  masked_mean_kernel<<<grid, 256, 0, ST>>>(x, ldx, y, ldy, T, C, len, bwd);
  return check_launch("masked_mean");
}
extern "C" int evk_dropout(const float* x, float* y, int64_t n, float p, const uint64_t* seed_offset,
                           uint64_t stream_id, evk_stream_t stream) {
  EVK_REQUIRE(x && y && seed_offset && p >= 0.f && p < 1.f, EVK_ERR_ARG, "dropout: bad arguments");
  if (n == 0) return EVK_OK;
  dropout_kernel<<<grid1d((n + 3) / 4), 256, 0, ST>>>(x, y, n, p, (const unsigned long long*)seed_offset, stream_id);
  return check_launch("dropout");
}
extern "C" int evk_randn(float* y, int64_t n, const uint64_t* seed_offset, uint64_t stream_id, evk_stream_t stream) {
  EVK_REQUIRE(y && seed_offset, EVK_ERR_ARG, "randn: null tensor");
  if (n == 0) return EVK_OK;
  randn_kernel<<<grid1d((n + 3) / 4), 256, 0, ST>>>(y, n, (const unsigned long long*)seed_offset, stream_id);
  return check_launch("randn");
}
extern "C" int evk_rand_slice_ids(int64_t* ids, const int32_t* len, int32_t B, int32_t seg, const uint64_t* seed_offset,
                                  uint64_t stream_id, evk_stream_t stream) {
  EVK_REQUIRE(ids && len && seed_offset && B >= 1, EVK_ERR_ARG, "rand_slice_ids: bad arguments");
  rand_slice_ids_kernel<<<cdiv(B, 128), 128, 0, ST>>>((long long*)ids, len, B, seg,
                                                      (const unsigned long long*)seed_offset, stream_id);
  return check_launch("rand_slice_ids");
}
extern "C" int evk_advance_rng(uint64_t* seed_offset, uint64_t inc, evk_stream_t stream) {
  EVK_REQUIRE(seed_offset, EVK_ERR_ARG, "advance_rng: null");
  advance_rng_kernel<<<1, 1, 0, ST>>>((unsigned long long*)seed_offset, inc);
  return check_launch("advance_rng");
}
