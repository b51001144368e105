// Band-split Roformer separation, inference only: BS-Roformer (uvr5/bs_roformer.py, lib_v5/vr_network/bs_roformer.py:327-553)
// and Mel-Band Roformer (uvr5/mel_band_roformer.py, lib_v5/vr_network/mel_band_roformer.py:244-478).  Their rotary, gated axial
// attention (evk_rope_attn_fwd) is in attn64.cu, the inverse STFT in stft.cu.  Here:
//   band_input_kernel     the STFT output gathered through a bin table into 'b t (f s c)' band order, each band's segment
//                         L2-normalised (BS-Roformer's table is the identity; a bin two mel bands share appears in both)
//   mask_avg_kernel       the band-major complex masks summed per (bin, channel) over the bands covering the bin, in ascending
//                         band order, and divided by the bin's band count (the reference's scatter_add_ / num_bands_per_freq)
//   row_norm_kernel       x / max(||x||, 1e-12) per row, times sqrt(C) * gamma when gamma is given (RMSNorm; without gamma
//                         the caller folds gamma * sqrt(dim) into the next Linear)
#include <math.h>

#include "evk_common.cuh"

namespace evk {
namespace {

// One CTA per (b, t): the row of cplx [(b S + s) T + t][NB][2] in shared memory as (f s c), then one warp per band.  Column c of
// band i (c in [2 S bo[i], 2 S bo[i+1])) is slot j = c / (2 S) of the bin table, channel and component c % (2 S).
__global__ void __launch_bounds__(256) band_input_kernel(const float2* __restrict__ cplx, int S, int T, int NB,
                                                         const int* __restrict__ bo, const int* __restrict__ fidx, int nb,
                                                         float* __restrict__ y, int ldy) {
  extern __shared__ float srow[];
  const int bt = blockIdx.x, b = bt / T, t = bt - b * T;
  for (int e = threadIdx.x; e < S * NB; e += blockDim.x) {
    const int f = e / S, s = e - f * S;
    const float2 v = cplx[((long long)(b * S + s) * T + t) * NB + f];
    srow[2 * e] = v.x;
    srow[2 * e + 1] = v.y;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, S2 = 2 * S;
  float* yr = y + (long long)bt * ldy;
  for (int i = warp; i < nb; i += nw) {
    const int c0 = S2 * bo[i], c1 = S2 * bo[i + 1];
    float ss = 0.f;
    for (int c = c0 + lane; c < c1; c += 32) {
      const int j = c / S2;
      const float v = srow[S2 * fidx[j] + (c - S2 * j)];
      ss += v * v;
    }
    const float den = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    for (int c = c0 + lane; c < c1; c += 32) {
      const int j = c / S2;
      yr[c] = srow[S2 * fidx[j] + (c - S2 * j)] / den;
    }
  }
}

// One thread per complex entry (row, f, s) of the mask: sum over the slots cov[co[f] .. co[f+1]) (ascending) of the GLU output's
// complex pair (j S + s), divided by the count.
__global__ void __launch_bounds__(256) mask_avg_kernel(const float* __restrict__ g, int ldg, const int* __restrict__ co,
                                                       const int* __restrict__ cov, int S, int NB, long long rows,
                                                       float* __restrict__ m, int ldm) {
  const long long per_row = (long long)S * NB, n = rows * per_row;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / per_row;
    const int fs = (int)(e - r * per_row), f = fs / S, s = fs - f * S;
    const float* gr = g + r * ldg;
    const int k0 = co[f], k1 = co[f + 1];
    float re = 0.f, im = 0.f;
    for (int k = k0; k < k1; ++k) {
      const float2 v = *reinterpret_cast<const float2*>(gr + 2 * (cov[k] * S + s));
      re += v.x;
      im += v.y;
    }
    const float cnt = (float)(k1 - k0);
    *reinterpret_cast<float2*>(m + r * ldm + 2 * fs) = make_float2(re / cnt, im / cnt);
  }
}

// one warp per row: y = x / max(||x||, 1e-12) (* scale * gamma) (x and y may be the same rows: each lane reads its columns
// before it writes them)
template <bool kGamma>
__global__ void __launch_bounds__(256) row_norm_kernel(const float* x, int ldx, const float* __restrict__ gamma, float* y, int ldy,
                                                       long long rows, int C, float scale) {
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* xr = x + r * ldx;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) ss += xr[c] * xr[c];
  const float den = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  float* yr = y + r * ldy;
  for (int c = lane; c < C; c += 32) {
    if constexpr (kGamma) yr[c] = xr[c] / den * scale * gamma[c];
    else yr[c] = xr[c] / den;
  }
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_band_input(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, const int32_t* band_off,
                              const int32_t* bins, int32_t n_bands, float* y, int32_t ldy, evk_stream_t stream) {
  EVK_REQUIRE(cplx && band_off && bins && y, EVK_ERR_ARG, "band_input: null tensor");
  EVK_REQUIRE(B > 0 && (S == 1 || S == 2) && T > 0 && n_bins > 0 && n_bands > 0 && ldy > 0, EVK_ERR_ARG,
              "band_input: bad sizes B=%d S=%d T=%d bins=%d bands=%d ldy=%d", B, S, T, n_bins, n_bands, ldy);
  const size_t smem = (size_t)2 * S * n_bins * sizeof(float);
  EVK_REQUIRE(smem <= 48 * 1024, EVK_ERR_UNSUPPORTED, "band_input: %d bins x %d channels do not fit shared memory", n_bins, S);
  EVK_REQUIRE((long long)B * T <= 0x7fffffff, EVK_ERR_ARG, "band_input: too many frames");
  band_input_kernel<<<(unsigned)(B * T), 256, smem, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(cplx), S, T, n_bins,
                                                                              band_off, bins, n_bands, y, ldy);
  return check_launch("band_input");
}

extern "C" int evk_melband_mask_avg(const float* g, int32_t ldg, const int32_t* cover_off, const int32_t* cover, int32_t S,
                                    int32_t n_bins, int64_t rows, float* mask, int32_t ld_mask, evk_stream_t stream) {
  EVK_REQUIRE(g && cover_off && cover && mask, EVK_ERR_ARG, "melband_mask_avg: null tensor");
  EVK_REQUIRE((S == 1 || S == 2) && n_bins > 0 && rows >= 0 && ld_mask >= 2 * S * n_bins && ldg > 0, EVK_ERR_ARG,
              "melband_mask_avg: bad sizes S=%d bins=%d ldg=%d ld_mask=%d", S, n_bins, ldg, ld_mask);
  EVK_REQUIRE((uintptr_t)g % 8 == 0 && (uintptr_t)mask % 8 == 0 && ldg % 2 == 0 && ld_mask % 2 == 0, EVK_ERR_ARG,
              "melband_mask_avg: g and mask rows must be 8-byte aligned");
  if (rows == 0) return EVK_OK;
  const long long blocks = (rows * S * n_bins + 255) / 256;
  mask_avg_kernel<<<(unsigned)(blocks < kNumSMs * 32 ? blocks : kNumSMs * 32), 256, 0, (cudaStream_t)stream>>>(
      g, ldg, cover_off, cover, S, n_bins, rows, mask, ld_mask);
  return check_launch("melband_mask_avg");
}

extern "C" int evk_row_norm(const float* x, int32_t ldx, const float* gamma, float* y, int32_t ldy, int64_t rows, int32_t C,
                            evk_stream_t stream) {
  EVK_REQUIRE(x && y && C > 0 && rows >= 0 && ldx >= C && ldy >= C, EVK_ERR_ARG, "row_norm: bad arguments");
  EVK_REQUIRE(x == y ? ldx == ldy : true, EVK_ERR_ARG, "row_norm: in place needs ldx == ldy");
  if (rows == 0) return EVK_OK;
  EVK_REQUIRE((rows + 7) / 8 <= 0x7fffffff, EVK_ERR_ARG, "row_norm: too many rows");
  const unsigned grid = (unsigned)((rows + 7) / 8);
  if (gamma)
    row_norm_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, gamma, y, ldy, rows, C, (float)sqrt((double)C));
  else
    row_norm_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, nullptr, y, ldy, rows, C, 1.f);
  return check_launch("row_norm");
}
