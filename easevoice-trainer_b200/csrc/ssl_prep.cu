// Loudness normalisation of Normalize._name2go (reference src/normalization/normalize.py:155-160) for a batch of zero-padded
// rows of 32 kHz samples, one CTA per row:
//   m    = max |a| over the row's samples (exact, so the reduction order cannot change it; a NaN sample makes m NaN, as numpy)
//   a32  = (a / m * c1) + c2 * a    -> int16 the way x86 numpy's astype("int16") converts: truncated to int32, low 16 bits kept
//   a32b = (a / m * c1b) + c2b * a  -> float32, the input of the 32 -> 16 kHz resampler
// Every operation is one correctly rounded float32 operation in the reference's order (no FMA contraction), so both outputs are
// bit-identical to numpy's.  Samples at or past the row's length are written as 0.
#include "evk_common.cuh"

namespace evk {
namespace {

constexpr int SN_THREADS = 1024;
// normalize.py:62-63 (maxx = 0.95, alpha = 0.5): numpy evaluates the products in float64 and applies them as float32 scalars
constexpr float SN_C1 = (float)(0.95 * 0.5 * 32768.0), SN_C2 = (float)((1.0 - 0.5) * 32768.0);
constexpr float SN_C1B = (float)(0.95 * 0.5 * 1145.14), SN_C2B = (float)((1.0 - 0.5) * 1145.14);

__global__ void __launch_bounds__(SN_THREADS) ssl_normalize_kernel(const float* __restrict__ a, int lda, const int* __restrict__ lens,
                                                                   int L, short* __restrict__ a32, int ld16, float* __restrict__ a32b,
                                                                   int ldb, int* __restrict__ status) {
  const int b = blockIdx.x;
  const int n = min(max(lens[b], 0), L);
  const float* x = a + (long long)b * lda;
  float m = 0.f;
  int nan = 0;
  for (int i = threadIdx.x; i < n; i += SN_THREADS) {
    const float v = fabsf(x[i]);
    nan |= v != v;
    m = fmaxf(m, v);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float red[SN_THREADS / 32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  nan = __syncthreads_or(nan);
  m = red[0];
#pragma unroll
  for (int w = 1; w < SN_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  if (nan) m = __int_as_float(0x7fffffff);
  // normalize.py:156-158: `tmp_max > 2.2` compares in float64 and skips the file (an infinite sample lands here too); m == 0
  // or a NaN sample makes every output NaN (0 / 0), which the reference's NaN check then rejects
  if (threadIdx.x == 0) status[b] = (double)m > 2.2 ? EVK_SSL_SKIP : (m > 0.f ? EVK_SSL_OK : EVK_SSL_NONFINITE);
  short* y16 = a32 + (long long)b * ld16;
  float* yb = a32b + (long long)b * ldb;
  for (int i = threadIdx.x; i < L; i += SN_THREADS) {
    if (i < n) {
      const float v = x[i], r = __fdiv_rn(v, m);
      // |a32| <= c1 + c2 * 2.2 < 2^31 on every row that is written, where cvt.rzi equals x86's cvttss2si
      y16[i] = (short)__float2int_rz(__fadd_rn(__fmul_rn(r, SN_C1), __fmul_rn(SN_C2, v)));
      yb[i] = __fadd_rn(__fmul_rn(r, SN_C1B), __fmul_rn(SN_C2B, v));
    } else {
      y16[i] = 0;
      yb[i] = 0.f;
    }
  }
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_ssl_normalize(const float* a, int32_t lda, const int32_t* lens, int32_t B, int32_t L, int16_t* a32, int32_t ld16,
                                 float* a32b, int32_t ldb, int32_t* status, evk_stream_t stream) {
  EVK_REQUIRE(a && lens && a32 && a32b && status && B >= 1 && L >= 1 && lda >= L && ld16 >= L && ldb >= L, EVK_ERR_ARG,
              "ssl_normalize: bad arguments");
  ssl_normalize_kernel<<<B, SN_THREADS, 0, (cudaStream_t)stream>>>(a, lda, lens, L, a32, ld16, a32b, ldb, status);
  return check_launch("ssl_normalize");
}
