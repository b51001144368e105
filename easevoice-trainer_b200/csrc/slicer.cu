// The device half of AudioService.slicer (reference src/service/audio.py:142-183, src/audiokit/slicer/slicer.py).
//
// evk_frame_rms: Slicer.get_rms for a ragged batch of recordings.  Frame t of a row is
//   sqrt(mean(x[t*hop - win/2 .. t*hop - win/2 + win)^2)),  zeros outside the row (pad_mode="constant").
// A row of n samples has 1 + (n + 2 (win/2) - win) / hop frames: 1 + n / hop for even win.  Frames overlap win / hop times,
// so the row is cut into hop-sized blocks in the frames' phase (block j starts at j*hop - win/2) and every sample is squared
// once: S[j] is the sum over block j, P[j] the sum over its first win % hop samples, and frame t = S[t] + ... +
// S[t + win/hop - 1] + P[t + win/hop].  When hop divides win, P is not computed.
// Squares and sums are float64 in a fixed order (lane-strided within a warp, then a butterfly), the mean and the square root
// are float64, and the result is rounded to float32 once: within 1 float32 ulp of the exact value whatever the grid, and a
// row gives the same bits alone and inside a batch.  A NaN or Inf sample propagates to the frames that cover it.
//
// evk_slice_normalize: the chunk loop of audio.py:171-178 for every chunk of every recording.  Pass 1 takes max |x| of each
// chunk (exact, so the order cannot change it) through an integer atomicMax on the bit pattern of |x|, in which every NaN
// is above every number, as in np.abs(chunk).max().  Pass 2 applies the reference's float32 operations one by one, without
// FMA contraction, and converts to int16 the way x86 numpy's astype does.  Both passes cut a chunk into tiles, so one long
// chunk spreads over the whole device.
//
// evk_fragment_int16: TTS.audio_postprocess for every synthesised sentence at once.  The same max pass, then one apply pass that
// divides by the max when it is above 1, scales by 32768, converts as above, writes each fragment at its place in the output
// order and the silent interval after it.
#include <limits.h>

#include "evk_common.cuh"

namespace evk {
namespace {

constexpr int RMS_THREADS = 256, RMS_FRAMES = 64, RMS_MAX_Q = 64;       // frames per CTA; win <= RMS_MAX_Q * hop
constexpr int RMS_SLOTS = RMS_FRAMES + RMS_MAX_Q + 1;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool PARTIAL>
__global__ void __launch_bounds__(RMS_THREADS) frame_rms_kernel(const float* __restrict__ x, long long ldx, const int* __restrict__ lens,
                                                                int win, int hop, float* __restrict__ rms, int T, int ldr) {
  __shared__ double S[RMS_SLOTS], P[RMS_SLOTS];
  const int b = blockIdx.y, t0 = blockIdx.x * RMS_FRAMES;
  const long long n = max(lens[b], 0);
  const long long last = n + 2 * (win / 2) - win;                       // start of the last window in the padded row
  const int frames = last < 0 ? 0 : (int)min((long long)T, 1 + last / hop);
  const int nf = min(RMS_FRAMES, T - t0);
  float* out = rms + (long long)b * ldr + t0;
  if (t0 >= frames) {                                                   // past the row's end
    for (int f = threadIdx.x; f < nf; f += RMS_THREADS) out[f] = 0.f;
    return;
  }
  const float* row = x + (long long)b * ldx;
  const int q = win / hop, rem = win - q * hop;
  const int slots = nf + q + (PARTIAL ? 1 : 0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = warp; j < slots; j += RMS_THREADS / 32) {
    const long long start = (long long)(t0 + j) * hop - win / 2;
    double s = 0.0, p = 0.0;
    if (start < n && start + hop > 0) {
#pragma unroll 4
      for (int i = lane; i < hop; i += 32) {
        const long long k = start + i;
        const double v = (k >= 0 && k < n) ? (double)row[k] : 0.0;
        s += v * v;
        if (PARTIAL && i < rem) p += v * v;
      }
      s = warp_sum_f64(s);
      if (PARTIAL) p = warp_sum_f64(p);
    }
    if (lane == 0) {
      S[j] = s;
      if (PARTIAL) P[j] = p;
    }
  }
  __syncthreads();
  for (int f = threadIdx.x; f < nf; f += RMS_THREADS) {
    float r = 0.f;
    if (t0 + f < frames) {
      double s = 0.0;
      for (int i = 0; i < q; ++i) s += S[f + i];
      if (PARTIAL) s += P[f + q];
      r = (float)sqrt(s / (double)win);
    }
    out[f] = r;
  }
}

constexpr int SL_THREADS = 256, SL_UNROLL = 8, SL_STEP = SL_THREADS * SL_UNROLL;

// x86 numpy's float32 -> int16 astype: cvttss2si to int32 (NaN and everything outside int32 become INT_MIN, whose low 16 bits
// are 0), then the low 16 bits
__device__ __forceinline__ short to_int16_x86(float s) {
  return (short)(fabsf(s) < 2147483648.f ? __float2int_rz(s) : INT_MIN);
}

// tile size for the longest of a set of ragged rows: at most 1024 tiles, of at least 8 * SL_STEP samples each
inline long long slice_tile_size(long long max_len) { return max(8LL, (long long)cdiv(cdiv(max_len, 1024), SL_STEP)) * SL_STEP; }

// tile blockIdx.x of chunk blockIdx.y -> the chunk's offset and [lo, hi) within the chunk
__device__ __forceinline__ void slice_tile(const long long* __restrict__ chunks, long long tile, long long& off, long long& lo,
                                           long long& hi) {
  off = chunks[2 * blockIdx.y];
  const long long len = max(chunks[2 * blockIdx.y + 1], 0LL);
  lo = min(len, (long long)blockIdx.x * tile);
  hi = min(len, lo + tile);
}

__global__ void __launch_bounds__(SL_THREADS) slice_max_kernel(const float* __restrict__ x, const long long* __restrict__ chunks,
                                                               long long tile, unsigned* __restrict__ mbits) {
  long long off, lo, hi;
  slice_tile(chunks, tile, off, lo, hi);
  if (lo >= hi) return;
  x += off;
  unsigned m = 0u;
  for (long long base = lo + threadIdx.x; base < hi; base += SL_STEP) {
#pragma unroll
    for (int u = 0; u < SL_UNROLL; ++u) {
      const long long i = base + (long long)u * SL_THREADS;
      if (i < hi) m = max(m, __float_as_uint(x[i]) & 0x7fffffffu);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ unsigned red[SL_THREADS / 32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 1; w < SL_THREADS / 32; ++w) m = max(m, red[w]);
    atomicMax(mbits + blockIdx.y, m);
  }
}

__global__ void __launch_bounds__(SL_THREADS) slice_apply_kernel(const float* __restrict__ x, const long long* __restrict__ chunks,
                                                                 long long tile, const unsigned* __restrict__ mbits, float c1, float c2,
                                                                 short* __restrict__ y, int* __restrict__ status) {
  long long off, lo, hi;
  slice_tile(chunks, tile, off, lo, hi);
  const float m = __uint_as_float(mbits[blockIdx.y]);
  if (blockIdx.x == 0 && threadIdx.x == 0)
    status[blockIdx.y] = m == 0.f ? EVK_SLICE_SILENT : (m < __int_as_float(0x7f800000) ? EVK_SLICE_OK : EVK_SLICE_NONFINITE);
  if (lo >= hi) return;
  x += off;
  y += off;
  const bool loud = m > 1.f;
  for (long long base = lo + threadIdx.x; base < hi; base += SL_STEP) {
#pragma unroll
    for (int u = 0; u < SL_UNROLL; ++u) {
      const long long i = base + (long long)u * SL_THREADS;
      if (i < hi) {
        const float v = x[i];
        const float c = loud ? __fdiv_rn(v, m) : v;                                   // audio.py:173-174, in place
        const float a = __fadd_rn(__fmul_rn(__fdiv_rn(c, m), c1), __fmul_rn(c2, c));  // audio.py:175: the old max again
        y[i] = to_int16_x86(__fmul_rn(a, 32767.f));
      }
    }
  }
}

// TTS.audio_postprocess (inference/tts.py:878-907) for fragment blockIdx.y: y[dst, dst + len) = int16(c * 32768) with
// c = m > 1 ? x / m : x, then y[dst + len, dst + len + gap) = 0.  Tiles of `tile` samples cover len + gap.
__global__ void __launch_bounds__(SL_THREADS) fragment_apply_kernel(const float* __restrict__ x, const long long* __restrict__ frags,
                                                                    const long long* __restrict__ dst, long long tile, long long gap,
                                                                    const unsigned* __restrict__ mbits, short* __restrict__ y) {
  const long long len = max(frags[2 * blockIdx.y + 1], 0LL), total = len + gap;
  const long long lo = min(total, (long long)blockIdx.x * tile), hi = min(total, lo + tile);
  if (lo >= hi) return;
  x += frags[2 * blockIdx.y];
  y += dst[blockIdx.y];
  const float m = __uint_as_float(mbits[blockIdx.y]);
  const bool loud = m > 1.f;
  for (long long base = lo + threadIdx.x; base < hi; base += SL_STEP) {
#pragma unroll
    for (int u = 0; u < SL_UNROLL; ++u) {
      const long long i = base + (long long)u * SL_THREADS;
      if (i < hi) {
        short k = 0;
        if (i < len) {
          const float v = x[i];
          k = to_int16_x86(__fmul_rn(loud ? __fdiv_rn(v, m) : v, 32768.f));
        }
        y[i] = k;
      }
    }
  }
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_frame_rms(const float* x, int64_t ldx, const int32_t* lens, int32_t B, int32_t win, int32_t hop, float* rms,
                             int32_t T, int32_t ldr, evk_stream_t stream) {
  EVK_REQUIRE(x && lens && rms && B >= 1 && B <= 65535 && hop >= 1 && win >= 1 && T >= 1 && ldr >= T && ldx >= 0, EVK_ERR_ARG,
              "frame_rms: bad arguments");
  EVK_REQUIRE(win / hop <= RMS_MAX_Q, EVK_ERR_ARG, "frame_rms: win %d is more than %d hops of %d", win, RMS_MAX_Q, hop);
  const dim3 grid(cdiv(T, RMS_FRAMES), B);
  if (win % hop)
    frame_rms_kernel<true><<<grid, RMS_THREADS, 0, (cudaStream_t)stream>>>(x, ldx, lens, win, hop, rms, T, ldr);
  else
    frame_rms_kernel<false><<<grid, RMS_THREADS, 0, (cudaStream_t)stream>>>(x, ldx, lens, win, hop, rms, T, ldr);
  return check_launch("frame_rms");
}

extern "C" int evk_slice_normalize(const float* x, const int64_t* chunks, int32_t n_chunks, int64_t max_len, float c1, float c2,
                                   int16_t* y, float* m, int32_t* status, evk_stream_t stream) {
  EVK_REQUIRE(x && chunks && y && m && status && n_chunks >= 1 && n_chunks <= 65535 && max_len >= 1, EVK_ERR_ARG,
              "slice_normalize: bad arguments");
  const long long tile = slice_tile_size(max_len);
  const dim3 grid(cdiv(max_len, tile), n_chunks);
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(m, 0, sizeof(float) * n_chunks, st) != cudaSuccess) return check_launch("slice_normalize (memset)");
  slice_max_kernel<<<grid, SL_THREADS, 0, st>>>(x, (const long long*)chunks, tile, (unsigned*)m);
  slice_apply_kernel<<<grid, SL_THREADS, 0, st>>>(x, (const long long*)chunks, tile, (const unsigned*)m, c1, c2, y, status);
  return check_launch("slice_normalize");
}

extern "C" int evk_fragment_int16(const float* x, const int64_t* frags, const int64_t* dst, int32_t n_frags, int64_t max_len,
                                  int64_t gap, int16_t* y, float* m, evk_stream_t stream) {
  EVK_REQUIRE(x && frags && dst && y && m && n_frags >= 1 && n_frags <= 65535 && max_len >= 1 && gap >= 0, EVK_ERR_ARG,
              "fragment_int16: bad arguments");
  const long long tile = slice_tile_size(max_len);
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(m, 0, sizeof(float) * n_frags, st) != cudaSuccess) return check_launch("fragment_int16 (memset)");
  slice_max_kernel<<<dim3(cdiv(max_len, tile), n_frags), SL_THREADS, 0, st>>>(x, (const long long*)frags, tile, (unsigned*)m);
  fragment_apply_kernel<<<dim3(cdiv(max_len + gap, tile), n_frags), SL_THREADS, 0, st>>>(
      x, (const long long*)frags, (const long long*)dst, tile, gap, (const unsigned*)m, y);
  return check_launch("fragment_int16");
}
