// Nearest-codeword search (exact fp32), loss reductions and the fused AdamW pass.
// Reference: core_vq.py:172-180; losses.py:7-61 + sovits.py:513; sovits.py:286-319,503-525 + commons.py:140-155.
#include "evk_common.cuh"

namespace evk {

// ---- exact fp32 NT GEMM: C[m][n] = sum_k A[m][k] * B[n][k]  (64x64 tile, 4x4 per thread) -------
// Token indices must not depend on TF32 rounding, so the distance GEMM stays on the fp32 pipe.
__global__ void __launch_bounds__(256) sgemm_nt_kernel(const float* __restrict__ A, int lda, const float* __restrict__ Bm,
                                                       int ldb, float* __restrict__ C, int ldc, int M, int N, int K) {
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, kk = i & 15;
      As[kk][r] = (m0 + r < M && k0 + kk < K) ? A[(long long)(m0 + r) * lda + k0 + kk] : 0.f;
      Bs[kk][r] = (n0 + r < N && k0 + kk < K) ? Bm[(long long)(n0 + r) * ldb + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) C[(long long)m * ldc + n] = acc[i][j];
    }
}

// codes[r] = argmax_k -((|x_r|^2 - 2 dot[r][k]) + |e_k|^2), lowest index on ties (core_vq.py:172-180)
__global__ void vq_argmax_kernel(const float* __restrict__ dots, int ldd, const float* __restrict__ x, int ldx,
                                 const float* __restrict__ embed, int lde, int K, int D, long long* __restrict__ codes,
                                 float* __restrict__ enorm /* [K] scratch, precomputed */) {
  __shared__ float red[33];
  __shared__ float bv[8];
  __shared__ int bi[8];
  const long long r = blockIdx.x;
  float xx = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) { float t = x[r * ldx + d]; xx += t * t; }
  xx = block_sum(xx, red);
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float dist = -((xx - 2.f * dots[r * ldd + k]) + enorm[k]);
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
    codes[r] = besti;
  }
}

__global__ void rownorm_sq_kernel(const float* __restrict__ e, int lde, int K, int D, float* __restrict__ out) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) { float t = e[(long long)k * lde + d]; s += t * t; }
  s = warp_sum(s);
  if (lane == 0) out[k] = s;
}

// ---- loss reductions -----------------------------------------------------------------------
__global__ void reduce_loss_kernel(int kind, const float* __restrict__ a, const float* __restrict__ b, long long n,
                                   float scale, float* __restrict__ out) {
  __shared__ float red[33];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = a[i];
    if (kind == 0) { const float t = 1.f - v; acc += t * t; }
    else if (kind == 1) acc += v * v;
    else acc += fabsf(v - b[i]);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) out[blockIdx.x] = acc * scale;      // per-block partial (ordered_sum adds them)
}

__global__ void reduce_loss_bwd_kernel(int kind, const float* __restrict__ a, const float* __restrict__ b, long long n,
                                       float scale, const float* __restrict__ gout, float* __restrict__ da) {
  const float g = gout[0] * scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = a[i];
    float d;
    if (kind == 0) d = -2.f * (1.f - v);
    else if (kind == 1) d = 2.f * v;
    else { const float t = v - b[i]; d = t > 0.f ? 1.f : (t < 0.f ? -1.f : 0.f); }
    da[i] = g * d;
  }
}

__global__ void kl_loss_kernel(const float* __restrict__ zp, int ldz, const float* __restrict__ lq, int ldq,
                               const float* __restrict__ mp, int ldm, const float* __restrict__ lp, int ldp, long long rows,
                               int T, int C, const int* __restrict__ len, float* __restrict__ out) {
  __shared__ float red[33];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * C; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    const long long bb = r / T;
    const int t = (int)(r - bb * T);
    if (len && t >= len[bb]) continue;
    const float d = zp[r * ldz + c] - mp[r * ldm + c], l = lp[r * ldp + c];
    acc += l - lq[r * ldq + c] - 0.5f + 0.5f * d * d * __expf(-2.f * l);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) out[blockIdx.x] = acc;             // per-block partial (ordered_sum adds them)
}

__global__ void kl_loss_bwd_kernel(const float* __restrict__ zp, int ldz, const float* __restrict__ lq, int ldq,
                                   const float* __restrict__ mp, int ldm, const float* __restrict__ lp, int ldp,
                                   long long rows, int T, int C, const int* __restrict__ len, const float* __restrict__ gout,
                                   float gscale, float* __restrict__ dzp, float* __restrict__ dlq, float* __restrict__ dmp,
                                   float* __restrict__ dlp, int ldg) {
  const float g = gout[0] * gscale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * C; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    const long long bb = r / T;
    const int t = (int)(r - bb * T);
    float a = 0.f, q = 0.f, p = 0.f;
    if (!(len && t >= len[bb])) {
      const float d = zp[r * ldz + c] - mp[r * ldm + c], e = __expf(-2.f * lp[r * ldp + c]);
      a = g * d * e;
      q = -g;
      p = g * (1.f - d * d * e);
    }
    dzp[r * ldg + c] = a;
    dmp[r * ldg + c] = -a;
    dlq[r * ldg + c] = q;
    dlp[r * ldg + c] = p;
  }
}

// ---- fused AdamW over a flat arena -----------------------------------------------------------
// hyper (device): [lr, step]  -- step is the 1-based AdamW step counter kept on the device (graph-replay safe);
// bias corrections 1 - beta^step are derived here in double precision.
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             long long n, const float* __restrict__ hyper, float lr_scale, float beta1, float beta2, float eps,
                             float wd, float grad_scale, float* __restrict__ gnorm_sq) {
  __shared__ float red[33];
  const float lr = hyper[0] * lr_scale;
  const double stepd = (double)hyper[1];
  const float bc1 = (float)(1.0 - pow((double)beta1, stepd)), bc2 = (float)(1.0 - pow((double)beta2, stepd));
  const float step = lr / bc1, isq = rsqrtf(bc2);
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gr = g[i] * grad_scale;
    acc += gr * gr;
    float pp = p[i] * (1.f - lr * wd);
    const float mm = beta1 * m[i] + (1.f - beta1) * gr;
    const float vv = beta2 * v[i] + (1.f - beta2) * gr * gr;
    pp -= step * mm / (sqrtf(vv) * isq + eps);
    p[i] = pp; m[i] = mm; v[i] = vv;
  }
  if (gnorm_sq) {
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) gnorm_sq[blockIdx.x] = acc;         // per-block partial (ordered_sum adds them)
  }
}

static inline dim3 g1(long long n) {
  long long g = (n + 255) / 256;
  if (g > (long long)kNumSMs * 16) g = (long long)kNumSMs * 16;
  if (g < 1) g = 1;
  return dim3((unsigned)g);
}

}  // namespace evk
using namespace evk;
#define ST ((cudaStream_t)stream)

extern "C" int evk_sgemm_nt_f32(const float* A, int32_t lda, const float* B, int32_t ldb, float* C, int32_t ldc,
                                int32_t M, int32_t N, int32_t K, evk_stream_t stream) {
  EVK_REQUIRE(A && B && C && M >= 1 && N >= 1 && K >= 1, EVK_ERR_ARG, "sgemm_nt: bad arguments");
  dim3 grid(cdiv(N, 64), cdiv(M, 64));
  EVK_REQUIRE(grid.y <= 65535, EVK_ERR_ARG, "sgemm_nt: M too large");
  sgemm_nt_kernel<<<grid, 256, 0, ST>>>(A, lda, B, ldb, C, ldc, M, N, K);
  return check_launch("sgemm_nt");
}

extern "C" int evk_vq_argmax(const float* dots, int32_t ldd, const float* x, int32_t ldx, const float* embed, int32_t lde,
                             int64_t rows, int32_t K, int32_t D, int64_t* codes, float* enorm_scratch,
                             evk_stream_t stream) {
  EVK_REQUIRE(dots && x && embed && codes && enorm_scratch, EVK_ERR_ARG, "vq_argmax: null tensor");
  if (rows == 0) return EVK_OK;
  rownorm_sq_kernel<<<cdiv(K, 8), 256, 0, ST>>>(embed, lde, K, D, enorm_scratch);
  int rc = check_launch("vq_rownorm");
  if (rc) return rc;
  vq_argmax_kernel<<<(unsigned)rows, 256, 0, ST>>>(dots, ldd, x, ldx, embed, lde, K, D, (long long*)codes, enorm_scratch);
  return check_launch("vq_argmax");
}

extern "C" int evk_reduce_loss(int32_t kind, const float* a, const float* b, int64_t n, float scale, float* out,
                               evk_stream_t stream) {
  EVK_REQUIRE(a && out && kind >= 0 && kind <= 2 && (kind != 2 || b), EVK_ERR_ARG, "reduce_loss: bad arguments");
  if (n == 0) return EVK_OK;
  const dim3 g = g1(n);
  Scratch part_buf(g.x, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "reduce_loss: scratch allocation failed");
  reduce_loss_kernel<<<g, 256, 0, ST>>>(kind, a, b, n, scale, part);
  if (int rc = check_launch("reduce_loss")) return rc;
  return ordered_sum(part, g.x, 1, 1, 1, out, 0, 0, ST);
}
extern "C" int evk_reduce_loss_bwd(int32_t kind, const float* a, const float* b, int64_t n, float scale,
                                   const float* gout, float* da, evk_stream_t stream) {
  EVK_REQUIRE(a && gout && da && kind >= 0 && kind <= 2 && (kind != 2 || b), EVK_ERR_ARG, "reduce_loss_bwd: bad arguments");
  if (n == 0) return EVK_OK;
  reduce_loss_bwd_kernel<<<g1(n), 256, 0, ST>>>(kind, a, b, n, scale, gout, da);
  return check_launch("reduce_loss_bwd");
}
extern "C" int evk_kl_loss(const float* z_p, int32_t ldz, const float* logs_q, int32_t ldq, const float* m_p, int32_t ldm,
                           const float* logs_p, int32_t ldp, int32_t B, int32_t T, int32_t C, const int32_t* len,
                           float* out, evk_stream_t stream) {
  EVK_REQUIRE(z_p && logs_q && m_p && logs_p && out, EVK_ERR_ARG, "kl_loss: null tensor");
  const long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  const dim3 g = g1(rows * C);
  Scratch part_buf(g.x, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "kl_loss: scratch allocation failed");
  kl_loss_kernel<<<g, 256, 0, ST>>>(z_p, ldz, logs_q, ldq, m_p, ldm, logs_p, ldp, rows, T, C, len, part);
  if (int rc = check_launch("kl_loss")) return rc;
  return ordered_sum(part, g.x, 1, 1, 1, out, 0, 0, ST);
}
extern "C" int evk_kl_loss_bwd(const float* z_p, int32_t ldz, const float* logs_q, int32_t ldq, const float* m_p,
                               int32_t ldm, const float* logs_p, int32_t ldp, int32_t B, int32_t T, int32_t C,
                               const int32_t* len, const float* gout, float gscale, float* dz_p, float* dlogs_q,
                               float* dm_p, float* dlogs_p, int32_t ldg, evk_stream_t stream) {
  EVK_REQUIRE(z_p && logs_q && m_p && logs_p && gout && dz_p && dlogs_q && dm_p && dlogs_p, EVK_ERR_ARG,
              "kl_loss_bwd: null tensor");
  const long long rows = (long long)B * T;
  if (rows * C == 0) return EVK_OK;
  kl_loss_bwd_kernel<<<g1(rows * C), 256, 0, ST>>>(z_p, ldz, logs_q, ldq, m_p, ldm, logs_p, ldp, rows, T, C, len, gout,
                                                   gscale, dz_p, dlogs_q, dm_p, dlogs_p, ldg);
  return check_launch("kl_loss_bwd");
}
__global__ void scalar_add_kernel(float* x, float v) { x[0] += v; }

extern "C" int evk_scalar_add(float* x, float v, evk_stream_t stream) {
  EVK_REQUIRE(x, EVK_ERR_ARG, "scalar_add: null");
  scalar_add_kernel<<<1, 1, 0, ST>>>(x, v);
  return check_launch("scalar_add");
}

extern "C" int evk_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* hyper, float lr_scale,
                              float beta1, float beta2, float eps, float wd, float grad_scale, float* gnorm_sq,
                              evk_stream_t stream) {
  EVK_REQUIRE(p && g && m && v && hyper, EVK_ERR_ARG, "adamw_flat: null tensor");
  if (n == 0) return EVK_OK;
  const dim3 gr = g1(n);
  Scratch part_buf(gnorm_sq ? gr.x : 0, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(!gnorm_sq || part, EVK_ERR_CUDA, "adamw_flat: scratch allocation failed");
  adamw_kernel<<<gr, 256, 0, ST>>>(p, g, m, v, n, hyper, lr_scale, beta1, beta2, eps, wd, grad_scale, part);
  if (int rc = check_launch("adamw_flat")) return rc;
  return gnorm_sq ? ordered_sum(part, gr.x, 1, 1, 1, gnorm_sq, 0, 0, ST) : EVK_OK;
}
