// UVR5 MDX23C (the TFC-TDF v3 U-Net, mdx23c.py), inference only, channels-last fp32 [B, H, W, C] activations with the
// spatial axes (time, frequency).  The 3x3, 1x1 and 2x2 stride-2 convolutions run on evk_conv2d_fwd, the instance norms on
// evk_instnorm_plane, the STFT / iSTFT on evk_stft_fwd / evk_istft.  Here:
//   tdf_kernel       the TDF Linear along the frequency axis: per (item, frame) slab Y[m][n] = sum_k A[m][k] X[k][n] (+ R),
//                    m, k frequencies (X rows strided by the pixel pitch), n channels.  The reduced axis is strided, so the
//                    slab is staged k-major into shared memory as it lies in HBM and read by TF32 mma.sync (whose B fragment
//                    takes either order from shared memory); wgmma would need it transposed first.  3xTF32 under
//                    evk_set_precise(1).  One fixed K order and no atomics: bit-reproducible and independent of the batch.
//   convt2x2         ConvTranspose2d(k = 2, stride = 2): four 1x1 convolutions, one per output phase (dy, dx), each writing
//                    every other pixel of every other output row straight into the destination (a decoder concat buffer).
//   mdx_front/back   the STFT <-> cac2cws / cws2cac layouts; mdx_add the residual adds and the `x * first_conv_out` product.
#include "evk_common.cuh"

namespace evk {
extern int g_precise;
namespace {

constexpr int TBM = 128, TBN = 64, TBK = 32, TLDA = TBK + 4, TLDB = TBN + 8;   // conflict-free fragment reads
constexpr int TSTAGES = 3, TNT = 256;
constexpr int TSLAB = TBM * TLDA + TBK * TLDB;
constexpr int TDF_SMEM = TSTAGES * TSLAB * 4;

struct TdfArgs {
  const float* a; const float* x; const float* r; float* y;
  long long x_zs, r_zs, y_zs;
  int ldx, ldr, ldy, M, N, K;
};

// stage K-slab k0: A [TBM][TLDA] (rows m, columns k) and X [TBK][TLDB] (rows k, columns n); outside the problem zero-filled
__device__ __forceinline__ void tdf_load(const TdfArgs& p, const float* xz, float* sA, float* sB, int k0, int m0, int n0) {
  const int tid = threadIdx.x;
  {
    const int kc = tid & 31, rr = tid >> 5;
    const int k = k0 + kc;
#pragma unroll 4
    for (int i = 0; i < TBM / 8; ++i) {
      const int m = m0 + rr + 8 * i;
      const bool ok = k < p.K && m < p.M;
      cp_async4(sA + (rr + 8 * i) * TLDA + kc, ok ? p.a + (long long)m * p.K + k : p.a, ok ? 4 : 0);
    }
  }
  {
    const int nc = tid & 63, rr = tid >> 6;
    const int n = n0 + nc;
#pragma unroll
    for (int i = 0; i < TBK / 4; ++i) {
      const int k = k0 + rr + 4 * i;
      const bool ok = k < p.K && n < p.N;
      cp_async4(sB + (rr + 4 * i) * TLDB + nc, ok ? xz + (long long)k * p.ldx + n : p.x, ok ? 4 : 0);
    }
  }
}

template <bool PR>
__global__ void __launch_bounds__(TNT, 2) tdf_kernel(TdfArgs p) {
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int m0 = blockIdx.x * TBM, n0 = blockIdx.y * TBN;
  const long long z = blockIdx.z;
  const float* xz = p.x + z * p.x_zs;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int nk = (p.K + TBK - 1) / TBK;
#pragma unroll
  for (int s = 0; s < TSTAGES - 1; ++s) {
    if (s < nk) tdf_load(p, xz, smem + s * TSLAB, smem + s * TSLAB + TBM * TLDA, s * TBK, m0, n0);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<TSTAGES - 2>();
    __syncthreads();
    {
      const int nx = kt + TSTAGES - 1, st = nx % TSTAGES;
      if (nx < nk) tdf_load(p, xz, smem + st * TSLAB, smem + st * TSLAB + TBM * TLDA, nx * TBK, m0, n0);
      cp_async_commit();
    }
    const float* As = smem + (kt % TSTAGES) * TSLAB;
    const float* Bs = As + TBM * TLDA;
    // 3xTF32: each slab is summed from zero and added to acc in fp32, as conv2d_fwd_kernel does
    float part[2][4][4];
    float (&sum)[2][4][4] = PR ? part : acc;
    if (PR) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.f;
    }
#pragma unroll
    for (int ks = 0; ks < TBK; ks += 8) {
      uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const float* q = As + (wm + mi * 16 + gq) * TLDA + ks + t;
        const float v[4] = {q[0], q[8 * TLDA], q[4], q[8 * TLDA + 4]};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          ah[mi][e] = f2tf32(v[e]);
          if (PR) al[mi][e] = f2tf32(v[e] - __uint_as_float(ah[mi][e]));
        }
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float* q = Bs + (ks + t) * TLDB + wn + ni * 8 + gq;
        const float v[2] = {q[0], q[4 * TLDB]};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          bh[ni][e] = f2tf32(v[e]);
          if (PR) bl[ni][e] = f2tf32(v[e] - __uint_as_float(bh[ni][e]));
        }
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          if (PR) {
            mma_tf32(sum[mi][ni], al[mi], bh[ni]);
            mma_tf32(sum[mi][ni], ah[mi], bl[ni]);
          }
          mma_tf32(sum[mi][ni], ah[mi], bh[ni]);
        }
    }
    if (PR) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[i][j][e] += part[i][j][e];
    }
  }
  cp_async_wait<0>();
  // rows wm + mi*16 + gq (+8), columns wn + ni*8 + 2t (+1); the residual is read and the output written by the same thread,
  // so r may be y (in place)
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm + mi * 16 + gq + 8 * h;
      if (m >= p.M) continue;
      float* yr = p.y + z * p.y_zs + (long long)m * p.ldy;
      const float* rr = p.r ? p.r + z * p.r_zs + (long long)m * p.ldr : nullptr;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n0 + wn + ni * 8 + 2 * t + e;
          if (n >= p.N) continue;
          float v = acc[mi][ni][2 * h + e];
          if (rr) v += rr[n];
          yr[n] = v;
        }
    }
}

template <bool PR>
int launch_tdf(const TdfArgs& p, int Z, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tdf_kernel<PR>, cudaFuncAttributeMaxDynamicSharedMemorySize, TDF_SMEM);
    EVK_REQUIRE(e == cudaSuccess, EVK_ERR_CUDA, "mdx_tdf: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  tdf_kernel<PR><<<dim3(cdiv(p.M, TBM), cdiv(p.N, TBN), Z), TNT, TDF_SMEM, st>>>(p);
  return check_launch("mdx_tdf");
}

// y[b, t, j, (s 2 + c) k + u] = cplx[b S + s, t, u F + j, c]   (cac2cws of the first k F bins, spatial axes (t, j))
__global__ void mdx_front_kernel(const float* __restrict__ cplx, int S, int T, int NB, int k, int F, float* __restrict__ y,
                                 int ldy, long long total) {
  const int D = 2 * S * k;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % D);
    long long q = i / D;
    const int j = (int)(q % F); q /= F;
    const int t = (int)(q % T);
    const int b = (int)(q / T);
    const int u = ch % k, sc = ch / k, c = sc & 1, s = sc >> 1;
    y[q * F * ldy + (long long)j * ldy + ch] = cplx[(((long long)(b * S + s) * T + t) * NB + u * F + j) * 2 + c];
  }
}

// cplx[(b nt + g) S + s, t, f, c] = f < k F ? x[b, t, f % F, g D + (s 2 + c) k + f / F] : 0   (cws2cac, zero bins above dim_f)
__global__ void mdx_back_kernel(const float* __restrict__ x, int ldx, int nt, int S, int T, int NB, int k, int F,
                                float* __restrict__ cplx, long long total) {
  const int D = 2 * S * k;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i % NB);
    long long q = i / NB;
    const int t = (int)(q % T); q /= T;
    const int s = (int)(q % S); q /= S;
    const int g = (int)(q % nt);
    const int b = (int)(q / nt);
    float2 v = make_float2(0.f, 0.f);
    if (f < k * F) {
      const float* px = x + (((long long)b * T + t) * F + f % F) * ldx + g * D + 2 * s * k + f / F;
      v = make_float2(px[0], px[k]);
    }
    reinterpret_cast<float2*>(cplx)[i] = v;
  }
}

// y = (a + b) * m (m nullable: 1) per (pixel, channel)
__global__ void mdx_add_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb,
                               const float* __restrict__ m, int ldm, float* __restrict__ y, int ldy, long long P, int C) {
  const long long total = P * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long p = i / C;
    float v = a[p * lda + c] + b[p * ldb + c];
    if (m) v *= m[p * ldm + c];
    y[p * ldy + c] = v;
  }
}

inline unsigned grid_of(long long total) {
  const long long g = (total + 255) / 256;
  return (unsigned)(g < 32LL * kNumSMs ? g : 32LL * kNumSMs);
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_mdx_tdf(const float* a, const float* x, int32_t ldx, int64_t x_zs, const float* r, int32_t ldr, int64_t r_zs,
                           float* y, int32_t ldy, int64_t y_zs, int32_t Z, int32_t M, int32_t N, int32_t K, evk_stream_t stream) {
  EVK_REQUIRE(a && x && y, EVK_ERR_ARG, "mdx_tdf: null tensor");
  EVK_REQUIRE(Z >= 1 && Z <= 65535 && M >= 1 && N >= 1 && K >= 1 && ldx >= N && ldy >= N && (!r || ldr >= N), EVK_ERR_ARG,
              "mdx_tdf: bad sizes Z=%d M=%d N=%d K=%d", Z, M, N, K);
  EVK_REQUIRE(cdiv(N, TBN) <= 65535, EVK_ERR_ARG, "mdx_tdf: too many channels");
  TdfArgs p{a, x, r, y, x_zs, r_zs, y_zs, ldx, ldr, ldy, M, N, K};
  return g_precise ? launch_tdf<true>(p, Z, (cudaStream_t)stream) : launch_tdf<false>(p, Z, (cudaStream_t)stream);
}

extern "C" int evk_convt2x2_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, float* y, int32_t y_pitch,
                                int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t N, evk_stream_t stream) {
  EVK_REQUIRE(x && w && y && B >= 1 && H >= 1 && W >= 1 && C >= 1 && N >= 1, EVK_ERR_ARG, "convt2x2: bad arguments");
  EVK_REQUIRE(x_bs == (int64_t)H * W * x_pitch && y_bs == 4ll * H * W * y_pitch && (long long)B * H <= 0x7fffffff, EVK_ERR_ARG,
              "convt2x2: the input and output planes must be dense in the batch (x_bs = H W x_pitch, y_bs = 4 H W y_pitch)");
  // phase (dy, dx): input row (b, i) is item b H + i of a [B H, 1, W] operand; its outputs are pixels 2 x + dx of output row
  // 2 i + dy, i.e. item stride 4 W y_pitch and pixel pitch 2 y_pitch from pixel (dy 2 W + dx)
  for (int dy = 0; dy < 2; ++dy)
    for (int dx = 0; dx < 2; ++dx)
      if (int rc = evk_conv2d_fwd(x, x_pitch, (int64_t)W * x_pitch, w + (long long)(dy * 2 + dx) * N * C, nullptr, nullptr,
                                  y + ((long long)dy * 2 * W + dx) * y_pitch, 2 * y_pitch, 4ll * W * y_pitch, B * H, 1, W, C, N, 1,
                                  1, 0, 0, 1, 1, EVK_C2_NONE, stream))
        return rc;
  return EVK_OK;
}

extern "C" int evk_mdx_front(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, int32_t k, int32_t F, float* y,
                             int32_t ldy, evk_stream_t stream) {
  EVK_REQUIRE(cplx && y && B >= 1 && S >= 1 && T >= 1 && k >= 1 && F >= 1 && (long long)k * F <= n_bins && ldy >= 2 * S * k,
              EVK_ERR_ARG, "mdx_front: bad sizes S=%d k=%d F=%d n_bins=%d ldy=%d", S, k, F, n_bins, ldy);
  const long long total = (long long)B * T * F * 2 * S * k;
  mdx_front_kernel<<<grid_of(total), 256, 0, (cudaStream_t)stream>>>(cplx, S, T, n_bins, k, F, y, ldy, total);
  return check_launch("mdx_front");
}

extern "C" int evk_mdx_back(const float* x, int32_t ldx, int32_t B, int32_t nt, int32_t S, int32_t T, int32_t n_bins, int32_t k,
                            int32_t F, float* cplx, evk_stream_t stream) {
  EVK_REQUIRE(x && cplx && B >= 1 && nt >= 1 && S >= 1 && T >= 1 && k >= 1 && F >= 1 && (long long)k * F <= n_bins &&
                  ldx >= 2 * S * k * nt,
              EVK_ERR_ARG, "mdx_back: bad sizes nt=%d S=%d k=%d F=%d n_bins=%d ldx=%d", nt, S, k, F, n_bins, ldx);
  const long long total = (long long)B * nt * S * T * n_bins;
  mdx_back_kernel<<<grid_of(total), 256, 0, (cudaStream_t)stream>>>(x, ldx, nt, S, T, n_bins, k, F, cplx, total);
  return check_launch("mdx_back");
}

extern "C" int evk_mdx_add(const float* a, int32_t lda, const float* b, int32_t ldb, const float* m, int32_t ldm, float* y,
                           int32_t ldy, int64_t P, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(a && b && y && P >= 1 && C >= 1 && lda >= C && ldb >= C && ldy >= C && (!m || ldm >= C), EVK_ERR_ARG,
              "mdx_add: bad arguments");
  mdx_add_kernel<<<grid_of(P * C), 256, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, m, ldm, y, ldy, P, C);
  return check_launch("mdx_add");
}
