// Front and back end of the UVR5 VR separators (SeparateVR.separate, uvr5/separate.py:103-196, lib_v5/vr_network/spec_utils.py)
// around the net: the per-band STFT written straight into the combined spectrogram, its normalised magnitudes, the
// polyphase resampler of the band loop, and the assembly of every band's half spectrum for the inverse STFT.
//   band STFT : librosa.stft(n_fft, hop, hann, center=True) of each band, cropped into combine_spectrograms' rows with the
//               pre-filter gains, plus the top band's high-end slice that mirroring reads.  Frames of any size the
//               mixed-radix core takes (stft_core.cuh): the UVR5 bands are 640, 320, 512 and 960.
//   magnitude : |x| / max|x| (SeparateVR.inference's x_mag_pre) and the coefficient; max is exact, so the two-stage
//               reduction is reproducible in any order.
//   resample  : scipy.signal.resample_poly's alignment (zero-prefixed filter, n_pre_remove, ceil(n up / down) outputs),
//               taps designed on the host.
//   assembly  : pred * exp(i angle(x)), x - that, mirroring and the fft_lp_filter / fft_hp_filter gains of
//               cmb_spectrogram_to_wave, for both outputs and both channels, into evk_istft's frame input.
#include "evk_common.cuh"
#include <math.h>

#include "stft_core.cuh"

namespace evk {

int stft_mr_tables(const float2** tw, const float** hann);      // stft.cu

namespace {

constexpr int VR_THREADS = 256;
constexpr int VR_MAX_BANDS = 4;
constexpr int VR_MAG_BLOCKS = 264;

struct VrBand {
  long long wav_off;          // band rows start at wav + wav_off, pitch ldw
  int L, ldw, N, hop, crop_start, crop_stop, row0;
};

struct VrStftP {
  const float* wav; VrBand band[VR_MAX_BANDS]; int n_bands, l, n_rows;
  const float* row_gain; float2* spec;
  int high_band, high_lo, high_h; float2* high;
  bool zero_pad;
  const float2* tw; const float* hann;
};

// grid (l frames, 2 n_bands): block (t, 2 b + c) transforms frame t of channel c of band b and scatters its crop range
__global__ void __launch_bounds__(VR_THREADS) vr_band_stft_kernel(const VrStftP p) {
  extern __shared__ __align__(16) uint8_t ssm[];
  const int t = blockIdx.x, b = blockIdx.y >> 1, c = blockIdx.y & 1;
  const VrBand& B = p.band[b];
  const int NH = B.N >> 1;
  float2* d0 = reinterpret_cast<float2*>(ssm);
  float2* d1 = d0 + NH;
  float2* sx = d1 + NH;
  const int tid = threadIdx.x;
  stft_load_phase_t(tid, VR_THREADS, p.wav + B.wav_off + (long long)c * B.ldw, B.L, t * B.hop - NH, B.N, B.N, p.hann, STFT_TAB_MR,
                    p.zero_pad, d0);
  __syncthreads();
  float2 *src = d0, *dst = d1;
  for (int Ns = 1; Ns < NH;) {
    Ns = stft_pass_r(tid, VR_THREADS, NH, Ns, stft_radix(NH, Ns), src, dst, p.tw, STFT_TAB_MR);
    __syncthreads();
    float2* tmp = src; src = dst; dst = tmp;
  }
  stft_untangle_phase_t(tid, VR_THREADS, B.N, src, p.tw, STFT_TAB_MR, sx);
  __syncthreads();
  for (int k = B.crop_start + tid; k < B.crop_stop; k += VR_THREADS) {
    const int r = B.row0 + k - B.crop_start;
    const float g = p.row_gain[r];
    const float2 x = sx[k];
    p.spec[((long long)c * p.n_rows + r) * p.l + t] = make_float2(x.x * g, x.y * g);
  }
  if (p.high && b == p.high_band)
    for (int i = tid; i < p.high_h; i += VR_THREADS) p.high[((long long)c * p.high_h + i) * p.l + t] = sx[p.high_lo + i];
}

// mag[i] = |spec[i]|; part[block] = max over the block's elements
__global__ void __launch_bounds__(VR_THREADS) vr_mag_max_kernel(const float2* __restrict__ spec, long long n, float* __restrict__ mag,
                                                                 float* __restrict__ part) {
  __shared__ float red[VR_THREADS];
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * VR_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * VR_THREADS) {
    const float2 x = spec[i];
    const float a = hypotf(x.x, x.y);
    mag[i] = a;
    m = fmaxf(m, a);
  }
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = VR_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

// coef = max(part); mag /= coef (0 / 0 = NaN for an all-zero input, as the reference's numpy)
__global__ void __launch_bounds__(VR_THREADS) vr_mag_norm_kernel(float* __restrict__ mag, long long n, const float* __restrict__ part,
                                                                  int n_part, float* __restrict__ coef) {
  __shared__ float red[VR_THREADS];
  float m = 0.f;
  for (int i = threadIdx.x; i < n_part; i += VR_THREADS) m = fmaxf(m, part[i]);
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = VR_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  const float cf = red[0];
  if (blockIdx.x == 0 && threadIdx.x == 0) *coef = cf;
  for (long long i = (long long)blockIdx.x * VR_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * VR_THREADS) mag[i] = mag[i] / cf;
}

// y[r][n] = sum over i ascending of x[r][i] h[(n + n_pre_remove) down - i up], the terms with the index inside [0, nh)
__global__ void vr_resample_poly_kernel(const float* __restrict__ x, int L, int ldx, const float* __restrict__ h, int nh, int up, int down,
                                        int n_pre_remove, float* __restrict__ y, int n_out, int ldy) {
  const int r = blockIdx.y;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < n_out; n += gridDim.x * blockDim.x) {
    const long long q = (long long)(n + n_pre_remove) * down;
    // i up <= q  and  q - i up < nh
    long long lo = q - nh + 1;
    lo = lo <= 0 ? 0 : (lo + up - 1) / up;
    long long hi = q / up;
    if (hi > L - 1) hi = L - 1;
    float acc = 0.f;
    for (long long i = lo; i <= hi; ++i) acc += x[(long long)r * ldx + i] * h[q - i * up];
    y[(long long)r * ldy + n] = acc;
  }
}

struct VrAsmBand {
  int N, crop_start, crop_stop, row0;
  long long gain_off, out_off;    // gains [N/2 + 1] at gains + gain_off; frames [4][l][N/2 + 1] complex at out + 2 out_off
};

struct VrAsmP {
  const float2* x; const float* pred; const float* pred_tta; const float* coef; int n_rows, l;
  const float2* high; int high_h, mirror_lo, top;
  VrAsmBand band[VR_MAX_BANDS]; int n_bands;
  const float* gains; float2* out;
};

__device__ __forceinline__ float2 vr_phase(float2 x) {
  float s, c;
  sincosf(atan2f(x.y, x.x), &s, &c);        // numpy's exp(1j * angle(x)): angle(0) = 0, so a zero bin has phase 1
  return make_float2(c, s);
}

// combined-spectrogram bin (c, r, t) of output sig: 0 = pred * phase(x) (the instruments), 1 = x - that (the vocals)
__device__ __forceinline__ float2 vr_out_bin(const VrAsmP& p, int sig, int c, int r, int t) {
  const long long i = ((long long)c * p.n_rows + r) * p.l + t;
  const float cf = *p.coef;
  const float pr = p.pred_tta ? (p.pred[i] + p.pred_tta[i]) * 0.5f * cf : p.pred[i] * cf;
  const float2 x = p.x[i], ph = vr_phase(x);
  const float2 y = make_float2(pr * ph.x, pr * ph.y);
  return sig == 0 ? y : make_float2(x.x - y.x, x.y - y.y);
}

// grid (l frames, n_bands): block (t, b) writes frame t of band b for the 4 rows (sig, c) -> out row 2 sig + c
__global__ void __launch_bounds__(VR_THREADS) vr_assemble_kernel(const VrAsmP p) {
  const int t = blockIdx.x, b = blockIdx.y;
  const VrAsmBand& B = p.band[b];
  const int NB = (B.N >> 1) + 1, max_bin = B.N >> 1;
  const bool top = (b == p.top) && p.high;
  for (int e = threadIdx.x; e < 4 * NB; e += VR_THREADS) {
    const int row = e / NB, k = e - row * NB, sig = row >> 1, c = row & 1;
    float2 v = make_float2(0.f, 0.f);
    if (top && k >= max_bin - p.high_h && k < max_bin) {
      // mirroring: i-th high-end bin against the flipped magnitude of rows [mirror_lo, mirror_lo + h) with its phase
      const int i = k - (max_bin - p.high_h);
      const float2 he = p.high[((long long)c * p.high_h + i) * p.l + t];
      const float2 m = vr_out_bin(p, sig, c, p.mirror_lo + p.high_h - 1 - i, t);
      const float mag = hypotf(m.x, m.y);
      const float2 ph = vr_phase(he);
      const float2 mirror = make_float2(mag * ph.x, mag * ph.y);
      v = (hypotf(he.x, he.y) <= hypotf(mirror.x, mirror.y)) ? he : mirror;
    } else if (k >= B.crop_start && k < B.crop_stop) {
      v = vr_out_bin(p, sig, c, B.row0 + k - B.crop_start, t);
    }
    const float g = p.gains[B.gain_off + k];
    p.out[B.out_off + ((long long)row * p.l + t) * NB + k] = make_float2(v.x * g, v.y * g);
  }
}

}  // namespace
}  // namespace evk

using namespace evk;

// bands: host int64 [n_bands][8] = (wav offset in floats, L, ldw, n_fft, hop, crop_start, crop_stop, first combined row)
extern "C" int evk_vr_band_stft(const float* wav, const int64_t* bands, int32_t n_bands, int32_t l, const float* row_gain, float* spec,
                                int32_t n_rows, int32_t high_band, int32_t high_lo, int32_t high_h, float* high, int32_t zero_pad,
                                evk_stream_t stream) {
  EVK_REQUIRE(wav && bands && row_gain && spec && n_bands >= 1 && n_bands <= VR_MAX_BANDS && l >= 1 && n_rows >= 1, EVK_ERR_ARG,
              "vr_band_stft: bad arguments");
  VrStftP p{};
  p.wav = wav; p.n_bands = n_bands; p.l = l; p.n_rows = n_rows; p.row_gain = row_gain; p.spec = reinterpret_cast<float2*>(spec);
  p.high_band = high_band; p.high_lo = high_lo; p.high_h = high_h; p.high = reinterpret_cast<float2*>(high); p.zero_pad = zero_pad != 0;
  int max_n = 0;
  for (int b = 0; b < n_bands; ++b) {
    const int64_t* d = bands + 8 * b;
    VrBand& B = p.band[b];
    B.wav_off = d[0]; B.L = (int)d[1]; B.ldw = (int)d[2]; B.N = (int)d[3]; B.hop = (int)d[4];
    B.crop_start = (int)d[5]; B.crop_stop = (int)d[6]; B.row0 = (int)d[7];
    EVK_REQUIRE(stft_mr_size_ok(B.N), EVK_ERR_UNSUPPORTED, "vr_band_stft: n_fft=%d must be an even divisor of %d in [16, 7680]", B.N,
                STFT_TAB_MR);
    EVK_REQUIRE(B.L >= 1 && B.ldw >= B.L && B.hop > 0 && 1 + B.L / B.hop >= l, EVK_ERR_ARG, "vr_band_stft: band %d has %d < %d frames", b,
                B.L >= 1 && B.hop > 0 ? 1 + B.L / B.hop : 0, l);
    EVK_REQUIRE(0 <= B.crop_start && B.crop_start <= B.crop_stop && B.crop_stop <= B.N / 2 + 1 &&
                    B.row0 + B.crop_stop - B.crop_start <= n_rows, EVK_ERR_ARG, "vr_band_stft: band %d crop out of range", b);
    max_n = max_n > B.N ? max_n : B.N;
  }
  EVK_REQUIRE(!high || (high_band >= 0 && high_band < n_bands && high_lo >= 0 && high_h >= 0 &&
                        high_lo + high_h <= p.band[high_band].N / 2 + 1), EVK_ERR_ARG, "vr_band_stft: bad high-end slice");
  if (int rc = stft_mr_tables(&p.tw, &p.hann)) return rc;
  const size_t smem = (size_t)(max_n / 2) * 16 + (size_t)(max_n / 2 + 1) * 8;
  static size_t attr = 48 * 1024;
  if (smem > attr) {
    if (cudaFuncSetAttribute(vr_band_stft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return check_launch("vr_band_stft_kernel");
    attr = smem;
  }
  vr_band_stft_kernel<<<dim3((unsigned)l, (unsigned)(2 * n_bands)), VR_THREADS, smem, (cudaStream_t)stream>>>(p);
  return check_launch("vr_band_stft_kernel");
}

extern "C" int evk_vr_mag_norm(const float* spec, int64_t n, float* mag, float* coef, evk_stream_t stream) {
  EVK_REQUIRE(spec && mag && coef && n > 0, EVK_ERR_ARG, "vr_mag_norm: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  Scratch part_buf(VR_MAG_BLOCKS, st);
  EVK_REQUIRE(part_buf.p, EVK_ERR_CUDA, "vr_mag_norm: scratch allocation failed");
  vr_mag_max_kernel<<<VR_MAG_BLOCKS, VR_THREADS, 0, st>>>(reinterpret_cast<const float2*>(spec), n, mag, part_buf.p);
  if (int rc = check_launch("vr_mag_max_kernel")) return rc;
  vr_mag_norm_kernel<<<VR_MAG_BLOCKS, VR_THREADS, 0, st>>>(mag, n, part_buf.p, VR_MAG_BLOCKS, coef);
  return check_launch("vr_mag_norm_kernel");
}

extern "C" int evk_resample_poly(const float* x, int32_t rows, int32_t L, int32_t ldx, const float* h, int32_t nh, int32_t up, int32_t down,
                                 int32_t n_pre_remove, float* y, int32_t n_out, int32_t ldy, evk_stream_t stream) {
  EVK_REQUIRE(x && h && y && rows >= 1 && rows <= 65535 && L >= 1 && ldx >= L && nh >= 1 && up >= 1 && down >= 1 && n_pre_remove >= 0 &&
                  n_out >= 1 && ldy >= n_out, EVK_ERR_ARG, "resample_poly: bad arguments");
  const int bx = cdiv(n_out, 256);
  vr_resample_poly_kernel<<<dim3((unsigned)(bx < 2048 ? bx : 2048), (unsigned)rows), 256, 0, (cudaStream_t)stream>>>(
      x, L, ldx, h, nh, up, down, n_pre_remove, y, n_out, ldy);
  return check_launch("vr_resample_poly_kernel");
}

// bands: host int64 [n_bands][6] = (n_fft, crop_start, crop_stop, first combined row, gain offset, output offset in complex elements)
extern "C" int evk_vr_assemble(const float* x, const float* pred, const float* pred_tta, const float* coef, int32_t n_rows, int32_t l,
                               const float* high, int32_t high_h, int32_t mirror_lo, int32_t top, const int64_t* bands, int32_t n_bands,
                               const float* gains, float* out, evk_stream_t stream) {
  EVK_REQUIRE(x && pred && coef && bands && gains && out && n_bands >= 1 && n_bands <= VR_MAX_BANDS && l >= 1, EVK_ERR_ARG,
              "vr_assemble: bad arguments");
  EVK_REQUIRE(!high || (top >= 0 && top < n_bands && high_h >= 0 && mirror_lo >= 0 && mirror_lo + high_h <= n_rows), EVK_ERR_ARG,
              "vr_assemble: bad mirroring rows");
  VrAsmP p{};
  p.x = reinterpret_cast<const float2*>(x); p.pred = pred; p.pred_tta = pred_tta; p.coef = coef; p.n_rows = n_rows; p.l = l;
  p.high = reinterpret_cast<const float2*>(high); p.high_h = high_h; p.mirror_lo = mirror_lo; p.top = top; p.n_bands = n_bands;
  p.gains = gains; p.out = reinterpret_cast<float2*>(out);
  for (int b = 0; b < n_bands; ++b) {
    const int64_t* d = bands + 6 * b;
    VrAsmBand& B = p.band[b];
    B.N = (int)d[0]; B.crop_start = (int)d[1]; B.crop_stop = (int)d[2]; B.row0 = (int)d[3]; B.gain_off = d[4]; B.out_off = d[5];
    EVK_REQUIRE(B.N >= 2 && 0 <= B.crop_start && B.crop_start <= B.crop_stop && B.crop_stop <= B.N / 2 + 1 &&
                    B.row0 + B.crop_stop - B.crop_start <= n_rows, EVK_ERR_ARG, "vr_assemble: band %d crop out of range", b);
    EVK_REQUIRE(!high || b != top || high_h <= B.N / 2, EVK_ERR_ARG, "vr_assemble: high end wider than the top band");
  }
  vr_assemble_kernel<<<dim3((unsigned)l, (unsigned)n_bands), VR_THREADS, 0, (cudaStream_t)stream>>>(p);
  return check_launch("vr_assemble_kernel");
}
