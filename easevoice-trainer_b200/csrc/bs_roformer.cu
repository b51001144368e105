// BS-Roformer separation (uvr5/bs_roformer.py, lib_v5/vr_network/bs_roformer.py:327-553), inference only; its rotary, gated
// axial attention (evk_rope_attn_fwd) is in attn64.cu:
//   band_input_kernel     the STFT output in the band-split operand layout 'b t (f s c)', each band's segment L2-normalised
//   row_l2norm_kernel     x / max(||x||, 1e-12) per row (every other RMSNorm; gamma * sqrt(dim) is folded into the next Linear)
#include "evk_common.cuh"

namespace evk {
namespace {

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
}  // namespace evk

using namespace evk;

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
