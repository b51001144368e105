// Attention pieces that are not plain GEMMs: masked softmax with the windowed relative-position key
// term, and the relative-position key/value terms themselves (window w => 2w+1 taps, shared across heads).
// Reference: attentions.py:243-292 (+ :312-365 skew helpers, replaced here by direct band indexing),
// modules.py:669-682 (MelStyleEncoder attention: -inf fill), mrte_model.py:54-59 (cross attention).
// Heads live inside the channel dim of channels-last tensors: q[b][t][h*dk + d].
#include "evk_common.cuh"

namespace evk {

// ---- softmax over keys, in place.  s = (S + relk_band) * scale, masked -> fill -------------
__global__ void attn_softmax_kernel(float* __restrict__ S, int lds, int H, int Tq, int Tk, float scale,
                                    const float* __restrict__ relk, int win, const int* __restrict__ qlen,
                                    const int* __restrict__ klen, float fill) {
  __shared__ float red[33];
  const long long row = blockIdx.x;                   // z*Tq + i
  const int z = (int)(row / Tq), i = (int)(row - (long long)z * Tq), b = z / H;
  float* s = S + row * lds;
  const int kl = klen ? min(klen[b], Tk) : Tk;
  const bool qdead = qlen && i >= qlen[b];
  const int W = 2 * win + 1;
  const float* rk = relk ? relk + row * W : nullptr;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    float v = s[j];
    if (rk) {
      const int r = j - i + win;
      if (r >= 0 && r < W) v += rk[r];
    }
    v *= scale;
    if (qdead || j >= kl) v = fill;
    s[j] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
    t = warp_max(t);
    if (threadIdx.x == 0) red[32] = t;
  }
  __syncthreads();
  mx = red[32];
  float sum = 0.f;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const float e = __expf(s[j] - mx);
    s[j] = e;
    sum += e;
  }
  sum = block_sum(sum, red);
  const float inv = 1.f / sum;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) s[j] *= inv;
}

// dS_raw = P * (dP - sum_j dP*P) * scale (in place on dP); drelk[row][r] = dS_raw[i][i + r - win]
__global__ void attn_softmax_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP, int lds, int Tq, int Tk, float scale,
                                        float* __restrict__ drelk, int win) {
  __shared__ float red[33];
  const long long row = blockIdx.x;
  const int i = (int)(row % Tq);
  const float* p = P + row * lds;
  float* d = dP + row * lds;
  float dot = 0.f;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) dot += p[j] * d[j];
  dot = block_sum(dot, red);
  const int W = 2 * win + 1;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const float v = p[j] * (d[j] - dot) * scale;
    d[j] = v;
    if (drelk) {
      const int r = j - i + win;
      if (r >= 0 && r < W) drelk[row * W + r] = v;
    }
  }
  if (drelk) {  // taps that fall outside [0, Tk) get zero
    for (int r = threadIdx.x; r < W; r += blockDim.x) {
      const int j = i + r - win;
      if (j < 0 || j >= Tk) drelk[row * W + r] = 0.f;
    }
  }
}

// rel[z][i][r] = sum_d q[b][i][h*dk+d] * E[r][d]          (thread per (z,i,r))
__global__ void relk_logits_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ E, int H, int T, int dk,
                                   int W, float* __restrict__ rel, long long total) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % W);
    const long long zi = idx / W;
    const int i = (int)(zi % T), z = (int)(zi / T), b = z / H, h = z - b * H;
    const float* qr = q + ((long long)b * T + i) * ldq + h * dk;
    const float* er = E + r * dk;
    float acc = 0.f;
    for (int d = 0; d < dk; ++d) acc = fmaf(qr[d], er[d], acc);
    rel[idx] = acc;
  }
}

// dq[b][i][h*dk+d] += sum_r drel[z][i][r] * E[r][d]       (thread per (z,i,d))
__global__ void relk_dq_kernel(const float* __restrict__ drel, const float* __restrict__ E, int H, int T, int dk, int W,
                               float* __restrict__ dq, int lddq, long long total) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(idx % dk);
    const long long zi = idx / dk;
    const int i = (int)(zi % T), z = (int)(zi / T), b = z / H, h = z - b * H;
    const float* dr = drel + zi * W;
    float acc = 0.f;
    for (int r = 0; r < W; ++r) acc = fmaf(dr[r], E[r * dk + d], acc);
    dq[((long long)b * T + i) * lddq + h * dk + d] += acc;
  }
}

// dE[r][d] += sum_{z,i} band[z][i][r] * x[b][i][h*dk+d]   (thread per (r,d), rows chunked over blocks; this kernel writes
// the partial of its row chunk to part[chunk][r*dk+d], ordered_sum adds the chunks in order)
// used for both dEk (band = drel, x = q) and dEv (band = P band, x = dOut)
__global__ void rel_dE_kernel(const float* __restrict__ band, const float* __restrict__ x, int ldx, int H, int T, int dk,
                              int W, float* __restrict__ dE, long long nrows, int rows_per_block) {
  const int rd = blockIdx.y * blockDim.x + threadIdx.x;
  if (rd >= W * dk) return;
  const int r = rd / dk, d = rd - r * dk;
  const int r0 = blockIdx.x * rows_per_block, r1 = (int)min(nrows, (long long)r0 + rows_per_block);   // nrows < 2^31 (checked by the host)
  float acc = 0.f;
  int i = r0 % T, z = r0 / T;
  for (int zi = r0; zi < r1; ++zi) {
    const int b = z / H, h = z - b * H;
    acc = fmaf(band[(long long)zi * W + r], x[((long long)b * T + i) * ldx + h * dk + d], acc);
    if (++i == T) { i = 0; ++z; }
  }
  dE[(long long)blockIdx.x * W * dk + rd] = acc;
}

// band[z][i][r] = P[z][i][i+r-win] (0 outside)            (to_band = 1)
// P[z][i][i+r-win] += band[z][i][r]                       (to_band = 0)
__global__ void attn_band_kernel(float* __restrict__ P, int lds, float* __restrict__ band, int Tq, int Tk, int win, int to_band,
                                 long long total) {
  const int W = 2 * win + 1;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % W);
    const long long row = idx / W;
    const int i = (int)(row % Tq);
    const int j = i + r - win;
    if (to_band) band[idx] = (j >= 0 && j < Tk) ? P[row * lds + j] : 0.f;
    else if (j >= 0 && j < Tk) P[row * lds + j] += band[idx];
  }
}

// out[b][i][h*dk+d] += sum_r band[z][i][r] * E[r][d]      (thread per (z,i,d))  -- relative value term
__global__ void relv_out_kernel(const float* __restrict__ band, const float* __restrict__ E, int H, int T, int dk, int W,
                                float* __restrict__ out, int ldo, long long total) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(idx % dk);
    const long long zi = idx / dk;
    const int i = (int)(zi % T), z = (int)(zi / T), b = z / H, h = z - b * H;
    const float* br = band + zi * W;
    float acc = 0.f;
    for (int r = 0; r < W; ++r) acc = fmaf(br[r], E[r * dk + d], acc);
    out[((long long)b * T + i) * ldo + h * dk + d] += acc;
  }
}

static inline dim3 g1(long long n) {
  long long g = (n + 255) / 256;
  if (g > (long long)kNumSMs * 32) g = (long long)kNumSMs * 32;
  if (g < 1) g = 1;
  return dim3((unsigned)g);
}

}  // namespace evk
using namespace evk;
#define ST ((cudaStream_t)stream)

extern "C" int evk_attn_softmax(float* S, int32_t lds, int32_t Z, int32_t H, int32_t Tq, int32_t Tk, float scale, const float* relk,
                                int32_t win, const int32_t* qlen, const int32_t* klen, float fill, evk_stream_t stream) {
  EVK_REQUIRE(S && Z >= 1 && H >= 1 && Tq >= 1 && Tk >= 1, EVK_ERR_ARG, "attn_softmax: bad arguments");
  const long long rows = (long long)Z * Tq;
  const int bs = Tk >= 256 ? 256 : (Tk >= 128 ? 128 : 64);
  attn_softmax_kernel<<<(unsigned)rows, bs, 0, ST>>>(S, lds, H, Tq, Tk, scale, relk, win, qlen, klen, fill);
  return check_launch("attn_softmax");
}
extern "C" int evk_attn_softmax_bwd(const float* P, float* dP, int32_t lds, int32_t Z, int32_t Tq, int32_t Tk, float scale,
                                    float* drelk, int32_t win, evk_stream_t stream) {
  EVK_REQUIRE(P && dP && Z >= 1, EVK_ERR_ARG, "attn_softmax_bwd: bad arguments");
  const long long rows = (long long)Z * Tq;
  const int bs = Tk >= 256 ? 256 : (Tk >= 128 ? 128 : 64);
  attn_softmax_bwd_kernel<<<(unsigned)rows, bs, 0, ST>>>(P, dP, lds, Tq, Tk, scale, drelk, win);
  return check_launch("attn_softmax_bwd");
}
extern "C" int evk_relk_logits(const float* q, int32_t ldq, const float* E, int32_t B, int32_t H, int32_t T, int32_t dk,
                               int32_t win, float* rel, evk_stream_t stream) {
  EVK_REQUIRE(q && E && rel, EVK_ERR_ARG, "relk_logits: null tensor");
  const int W = 2 * win + 1;
  const long long total = (long long)B * H * T * W;
  if (!total) return EVK_OK;
  relk_logits_kernel<<<g1(total), 256, 0, ST>>>(q, ldq, E, H, T, dk, W, rel, total);
  return check_launch("relk_logits");
}
extern "C" int evk_relk_bwd(const float* drel, const float* q, int32_t ldq, const float* E, int32_t B, int32_t H,
                            int32_t T, int32_t dk, int32_t win, float* dq, int32_t lddq, float* dE,
                            evk_stream_t stream) {
  EVK_REQUIRE(drel && q && E && dq && dE, EVK_ERR_ARG, "relk_bwd: null tensor");
  const int W = 2 * win + 1;
  const long long nrows = (long long)B * H * T;
  if (!nrows) return EVK_OK;
  relk_dq_kernel<<<g1(nrows * dk), 256, 0, ST>>>(drel, E, H, T, dk, W, dq, lddq, nrows * dk);
  int rc = check_launch("relk_dq");
  if (rc) return rc;
  EVK_REQUIRE(nrows < 0x7fffffffLL, EVK_ERR_ARG, "relk_bwd: too many rows");
  const int rpb = 32;
  dim3 grid(cdiv(nrows, rpb), cdiv(W * dk, 128));
  Scratch part_buf((long long)grid.x * W * dk, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "relk_bwd: scratch allocation failed");
  rel_dE_kernel<<<grid, 128, 0, ST>>>(drel, q, ldq, H, T, dk, W, part, nrows, rpb);
  if (int rc2 = check_launch("relk_dE")) return rc2;
  return ordered_sum(part, grid.x, 1, 1, W * dk, dE, 0, 0, ST);
}
extern "C" int evk_attn_band(float* P, int32_t lds, float* band, int32_t Z, int32_t Tq, int32_t Tk, int32_t win, int32_t to_band,
                             evk_stream_t stream) {
  EVK_REQUIRE(P && band, EVK_ERR_ARG, "attn_band: null tensor");
  const long long total = (long long)Z * Tq * (2 * win + 1);
  if (!total) return EVK_OK;
  attn_band_kernel<<<g1(total), 256, 0, ST>>>(P, lds, band, Tq, Tk, win, to_band, total);
  return check_launch("attn_band");
}
extern "C" int evk_relv_out(const float* band, const float* E, int32_t B, int32_t H, int32_t T, int32_t dk, int32_t win,
                            float* out, int32_t ldo, evk_stream_t stream) {
  EVK_REQUIRE(band && E && out, EVK_ERR_ARG, "relv_out: null tensor");
  const long long total = (long long)B * H * T * dk;
  if (!total) return EVK_OK;
  relv_out_kernel<<<g1(total), 256, 0, ST>>>(band, E, H, T, dk, 2 * win + 1, out, ldo, total);
  return check_launch("relv_out");
}
// dband[z][i][r] = sum_d dOut[b][i][h*dk+d] * E[r][d]  (== relk_logits with q := dOut);  dE via rel_dE
extern "C" int evk_relv_bwd(const float* band, const float* dout, int32_t lddo, const float* E, int32_t B, int32_t H,
                            int32_t T, int32_t dk, int32_t win, float* dband, float* dE, evk_stream_t stream) {
  EVK_REQUIRE(band && dout && E && dband && dE, EVK_ERR_ARG, "relv_bwd: null tensor");
  const int W = 2 * win + 1;
  const long long nrows = (long long)B * H * T;
  if (!nrows) return EVK_OK;
  relk_logits_kernel<<<g1(nrows * W), 256, 0, ST>>>(dout, lddo, E, H, T, dk, W, dband, nrows * W);
  int rc = check_launch("relv_dband");
  if (rc) return rc;
  EVK_REQUIRE(nrows < 0x7fffffffLL, EVK_ERR_ARG, "relv_bwd: too many rows");
  const int rpb = 32;
  dim3 grid(cdiv(nrows, rpb), cdiv(W * dk, 128));
  Scratch part_buf((long long)grid.x * W * dk, ST);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "relv_bwd: scratch allocation failed");
  rel_dE_kernel<<<grid, 128, 0, ST>>>(band, dout, lddo, H, T, dk, W, part, nrows, rpb);
  if (int rc2 = check_launch("relv_dE")) return rc2;
  return ordered_sum(part, grid.x, 1, 1, W * dk, dE, 0, 0, ST);
}
