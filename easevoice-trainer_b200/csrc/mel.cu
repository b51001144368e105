// Fused mel front end, fast path of the training configuration (n_fft = win = 2048, center=False): reflect-pad -> Hann ->
// 2048-point real FFT -> sqrt(re^2+im^2+1e-6) -> sparse Slaney filterbank -> log(clamp(., 1e-5)), one WARP per frame with the
// whole 1024-point complex FFT of the even/odd-packed frame in registers (fp32: the parity oracle is torch.stft in fp32).
// Every other (n_fft, hop, win, padding) and the adjoint live in stft.cu.
// Reference: src/easevoice/module/mel_processing.py:40-142.
#include "evk_common.cuh"
#include <math.h>

namespace evk {

constexpr int NFFT = 2048;
constexpr int NH = NFFT / 2;      // complex FFT length
constexpr int NBIN = NH + 1;      // 1025

__device__ float2 g_tw[NFFT];     // e^{-2 pi i k / 2048}
__device__ float g_hann[NFFT];    // periodic Hann
__device__ float2 g_tw32[32 * 32]; // [k1][t] = e^{-2 pi i t k1 / 1024}: inter-stage twiddles of the 32 x 32 warp FFT
static bool g_tables_ready = false;

int mel_init_tables() {
  if (g_tables_ready) return EVK_OK;
  static float2 tw[NFFT];
  static float hw[NFFT];
  for (int i = 0; i < NFFT; ++i) {
    double a = 2.0 * M_PI * (double)i / (double)NFFT;
    tw[i] = make_float2((float)cos(a), (float)(-sin(a)));
    hw[i] = (float)(0.5 - 0.5 * cos(a));
  }
  if (cudaMemcpyToSymbol(g_tw, tw, sizeof(tw)) != cudaSuccess) return EVK_ERR_CUDA;
  if (cudaMemcpyToSymbol(g_hann, hw, sizeof(hw)) != cudaSuccess) return EVK_ERR_CUDA;
  static float2 t32[32 * 32];
  for (int k1 = 0; k1 < 32; ++k1)
    for (int t = 0; t < 32; ++t) {
      double a = 2.0 * M_PI * (double)((t * k1) % 1024) / 1024.0;
      t32[k1 * 32 + t] = make_float2((float)cos(a), (float)(-sin(a)));
    }
  if (cudaMemcpyToSymbol(g_tw32, t32, sizeof(t32)) != cudaSuccess) return EVK_ERR_CUDA;
  g_tables_ready = true;
  return EVK_OK;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

__device__ __forceinline__ int reflect_idx(int i, int L) {
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  return i;
}

// ------------------------------------------------------------------------------------------------------------
// Warp-per-frame variant (the fast path): the 1024-point complex FFT of the even/odd packed frame is computed as
// 32 x 32 with all data in registers -- each lane runs a 32-point radix-2 FFT on its own registers (compile-time
// indices, compile-time twiddles), the warp transposes through shared memory once, each lane runs a second
// 32-point FFT.  No block-wide barrier, 8 frames per CTA, every global access coalesced.
// ------------------------------------------------------------------------------------------------------------
constexpr int MEL_WPB = 6;
constexpr int MEL_WARP_SMEM = 32 * 33 * 8 + (NBIN + 3) * 4;   // 12 560 B per warp
constexpr int MEL_FB_MAX = 2064;                                          // filterbank non-zeros staged in smem (2 016 for 128 Slaney mels)
// twiddles (2 tables) + CSR val (f32) / idx (u16) / ptr + the first half of the (symmetric) Hann window
constexpr int MEL_TAB_SMEM = 32 * 32 * 8 + (NH + 8) * 8 + MEL_FB_MAX * 4 + MEL_FB_MAX * 2 + 144 * 4 + (NH + 4) * 4;

__host__ __device__ constexpr int brev5(int k) {
  return ((k & 1) << 4) | ((k & 2) << 2) | (k & 4) | ((k & 8) >> 2) | ((k & 16) >> 4);
}

// cos(2 pi k / 32), sin(2 pi k / 32), k = 0..15
__device__ constexpr float C32[16] = {1.f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                                      0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f,
                                      0.19509032201612825f, 0.f, -0.19509032201612825f, -0.38268343236508977f,
                                      -0.55557023301960218f, -0.70710678118654752f, -0.83146961230254524f,
                                      -0.92387953251128674f, -0.98078528040323043f};
__device__ constexpr float S32[16] = {0.f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f,
                                      0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f,
                                      0.98078528040323043f, 1.f, 0.98078528040323043f, 0.92387953251128674f,
                                      0.83146961230254524f, 0.70710678118654752f, 0.55557023301960218f,
                                      0.38268343236508977f, 0.19509032201612825f};

// in-place 32-point DIF FFT on registers; X[k] ends up in element brev5(k)
__device__ __forceinline__ void fft32_regs(float (&xr)[32], float (&xi)[32]) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
#pragma unroll
    for (int blk = 0; blk < 32; blk += 2 * half) {
#pragma unroll
      for (int j = 0; j < half; ++j) {
        const int i0 = blk + j, i1 = i0 + half;
        const int tw = j * (16 / half);                       // exponent of W_32 (compile-time after unrolling)
        const float ar = xr[i0], ai = xi[i0], br = xr[i1], bi = xi[i1];
        xr[i0] = ar + br; xi[i0] = ai + bi;
        const float dr = ar - br, di = ai - bi;
        if (tw == 0) { xr[i1] = dr; xi[i1] = di; }
        else if (tw == 8) { xr[i1] = di; xi[i1] = -dr; }     // * (-i)
        else {                                                 // (dr + i di)(c - i s)
          xr[i1] = fmaf(dr, C32[tw], di * S32[tw]);
          xi[i1] = fmaf(di, C32[tw], -dr * S32[tw]);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(MEL_WPB * 32, 2) mel_fwd_warp_kernel(
    const float* __restrict__ wav, const int* __restrict__ lens, int Lmax, int ldw, int T, long long nframes, int hop, int n_mels,
    const int* __restrict__ fb_ptr, const int* __restrict__ fb_idx, const float* __restrict__ fb_val,
    float* __restrict__ spec, int ld_spec, float* __restrict__ mel, int ld_mel, float* __restrict__ cplx) {
  // persistent CTA: the three lookup tables are staged in shared memory once (the 200 KB of per-warp buffers leave
  // almost no L1, so table reads from global memory would otherwise go to L2 on every frame)
  extern __shared__ __align__(16) uint8_t msm[];
  float2* s_tw32 = reinterpret_cast<float2*>(msm);
  float2* s_tw = reinterpret_cast<float2*>(msm + 32 * 32 * 8);
  float* s_fval = reinterpret_cast<float*>(msm + 32 * 32 * 8 + (NH + 8) * 8);
  int* s_fptr = reinterpret_cast<int*>(s_fval + MEL_FB_MAX);
  float* s_hann = reinterpret_cast<float*>(s_fptr + 144);     // w[0 .. 1024]; w[n] = w[2048 - n] above
  unsigned short* s_fidx = reinterpret_cast<unsigned short*>(s_hann + NH + 4);
  uint8_t* wsm = msm + MEL_TAB_SMEM;                           // per warp: float2[32*33] transpose buffer + float[NBIN+3]
  for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x) s_tw32[i] = g_tw32[i];
  for (int i = threadIdx.x; i <= NH; i += blockDim.x) { s_tw[i] = g_tw[i]; s_hann[i] = g_hann[i]; }
  if (mel) {
    const int nnz = fb_ptr[n_mels];
    for (int i = threadIdx.x; i < nnz; i += blockDim.x) { s_fval[i] = fb_val[i]; s_fidx[i] = (unsigned short)fb_idx[i]; }
    for (int i = threadIdx.x; i <= n_mels; i += blockDim.x) s_fptr[i] = fb_ptr[i];
  }
  __syncthreads();
  const int w = threadIdx.x >> 5, t = threadIdx.x & 31;
  const int padc = (NFFT - hop) / 2;
  // A frame whose 2048 samples are interior and 16-byte aligned is staged through the warp's transpose buffer with cp.async
  // (one round trip, no registers held while it flies; ncu had the register-limited batches of direct loads as the top stall,
  // long_scoreboard 36 %), and the NEXT frame of this warp is put in flight as soon as the buffer is free again (after the
  // untangle pass), under the filterbank phase.
  auto stageable = [&](long long fr, const float*& src) -> bool {
    if (fr >= nframes) return false;
    const int bb = (int)(fr / T), ff = (int)(fr - (long long)bb * T);
    const int ss = ff * hop - padc;
    const int LL = lens ? min(lens[bb], Lmax) : Lmax;
    if (LL + 2 * padc < NFFT || ff >= (LL + 2 * padc - NFFT) / hop + 1) return false;
    src = wav + (long long)bb * ldw + ss;
    return ss >= 0 && ss + NFFT <= LL && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  };
  auto stage_issue = [&](const float* src, float* dst) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = (i * 32 + t) * 4;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(dst + c)), "l"(src + c));
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
  };
  long long staged = -1;                                        // frame whose samples are in flight / resident in this warp's buffer
  for (long long frame = (long long)blockIdx.x * MEL_WPB + w; frame < nframes; frame += (long long)gridDim.x * MEL_WPB) {
  const int b = (int)(frame / T), f = (int)(frame - (long long)b * T);
  const int pad = (NFFT - hop) / 2, s0 = f * hop - pad;
  const float* wv = wav + (long long)b * ldw;
  // per-row length: the reflection sits at the row's OWN end (the reference runs spectrogram_torch per utterance,
  // data_utils.py:119-128) and frames past the row's own count hold what the zero-padded collate holds
  const int L = lens ? min(lens[b], Lmax) : Lmax;
  if (f >= (L + 2 * pad - NFFT) / hop + 1 || L + 2 * pad < NFFT) {
    for (int k = t; k < NBIN; k += 32) {
      if (spec) spec[frame * ld_spec + k] = 0.f;
      if (cplx) reinterpret_cast<float2*>(cplx)[frame * NBIN + k] = make_float2(0.f, 0.f);
    }
    if (mel)
      for (int mm = t; mm < n_mels; mm += 32) mel[frame * ld_mel + mm] = logf(1e-5f);
    continue;
  }
  float xr[32], xi[32];
  float2* z = reinterpret_cast<float2*>(wsm + (size_t)w * MEL_WARP_SMEM);
  const float* fsrc = nullptr;
  const bool can_stage = stageable(frame, fsrc);
  if (can_stage) {
    if (staged != frame) stage_issue(fsrc, reinterpret_cast<float*>(z));
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncwarp();
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) {                          // z[m] = (x[2m] w[2m], x[2m+1] w[2m+1]), m = 32 n1 + t
      const int m = 32 * n1 + t;
      const float2 v = z[m];
      float2 hw;
      if (n1 < 16) hw = *reinterpret_cast<const float2*>(&s_hann[2 * m]);
      else hw = make_float2(s_hann[NFFT - 2 * m], s_hann[NFFT - 1 - 2 * m]);
      xr[n1] = v.x * hw.x;
      xi[n1] = v.y * hw.y;
    }
    __syncwarp();                                              // every lane has its samples: the buffer becomes the transpose tile
  } else {
    const bool interior = (s0 >= 0) && (s0 + NFFT <= L) && (((s0 & 1) == 0) && ((reinterpret_cast<uintptr_t>(wv) & 7) == 0));
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) {
      const int m = 32 * n1 + t;
      const float2 hw = *reinterpret_cast<const float2*>(&g_hann[2 * m]);
      float2 v;
      if (interior) v = *reinterpret_cast<const float2*>(wv + s0 + 2 * m);
      else v = make_float2(wv[reflect_idx(s0 + 2 * m, L)], wv[reflect_idx(s0 + 2 * m + 1, L)]);
      xr[n1] = v.x * hw.x;
      xi[n1] = v.y * hw.y;
    }
  }
  fft32_regs(xr, xi);                                          // A[k1][n2 = t] in element brev5(k1)
#pragma unroll
  for (int k1 = 0; k1 < 32; ++k1) {                            // inter-stage twiddle, then transpose through smem
    const float2 tw = s_tw32[k1 * 32 + t];
    const float ar = xr[brev5(k1)], ai = xi[brev5(k1)];
    z[k1 * 33 + t] = make_float2(ar * tw.x - ai * tw.y, ar * tw.y + ai * tw.x);
  }
  __syncwarp();
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) {                            // lane t now owns k1 = t
    const float2 v = z[t * 33 + n2];
    xr[n2] = v.x; xi[n2] = v.y;
  }
  __syncwarp();
  fft32_regs(xr, xi);                                          // Z[t + 32 k2] in element brev5(k2)
#pragma unroll
  for (int k2 = 0; k2 < 32; ++k2) z[t + 32 * k2] = make_float2(xr[brev5(k2)], xi[brev5(k2)]);
  __syncwarp();
  float* mg = reinterpret_cast<float*>(wsm + (size_t)w * MEL_WARP_SMEM + 32 * 33 * sizeof(float2));
  float2* cp = cplx ? reinterpret_cast<float2*>(cplx) + frame * NBIN : nullptr;
#pragma unroll
  for (int j = 0; j <= 32; ++j) {                              // real-FFT untangle: bins k = t + 32 j (+ bin 1024)
    const int k = t + 32 * j;
    if (j == 32 && t != 0) break;
    const float2 zk = (j < 32) ? make_float2(xr[brev5(j & 31)], xi[brev5(j & 31)]) : z[0];
    float2 zc = z[(NH - k) & (NH - 1)];
    zc.y = -zc.y;
    const float2 sm = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
    const float2 dd = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
    const float2 tw = s_tw[k];
    const float2 tt = cmul(tw, dd);
    const float2 X = make_float2(sm.x + tt.y, sm.y - tt.x);
    const float m = sqrtf(X.x * X.x + X.y * X.y + 1e-6f);
    mg[k] = m;
    if (spec) spec[frame * ld_spec + k] = m;
    if (cp) cp[k] = X;
  }
  __syncwarp();
  {                                                            // the transpose tile is free: put this warp's next frame in flight
    const long long nf = frame + (long long)gridDim.x * MEL_WPB;
    const float* nsrc = nullptr;
    if (stageable(nf, nsrc)) { stage_issue(nsrc, reinterpret_cast<float*>(z)); staged = nf; }
  }
  if (mel) {                                                   // sparse filterbank, CSR by mel row staged in shared memory
    for (int mm = t; mm < n_mels; mm += 32) {
      float acc = 0.f;
      const int e1 = s_fptr[mm + 1];
      for (int e = s_fptr[mm]; e < e1; ++e) acc = fmaf(s_fval[e], mg[s_fidx[e]], acc);
      mel[frame * ld_mel + mm] = logf(fmaxf(acc, 1e-5f));
    }
  }
  __syncwarp();                                                // the per-warp buffers are reused by the next frame
  }
}

__global__ void spec_to_mel_kernel(const float* __restrict__ spec, long long rows, int ld_spec, int n_mels,
                                   const int* __restrict__ fb_ptr, const int* __restrict__ fb_idx,
                                   const float* __restrict__ fb_val, float* __restrict__ mel, int ld_mel) {
  const long long row = blockIdx.x;
  const float* s = spec + row * ld_spec;
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    float acc = 0.f;
    for (int e = fb_ptr[m]; e < fb_ptr[m + 1]; ++e) acc = fmaf(fb_val[e], s[fb_idx[e]], acc);
    mel[row * ld_mel + m] = logf(fmaxf(acc, 1e-5f));
  }
}

}  // namespace evk
using namespace evk;

static int g_mel_variant = 1;      // 1: warp-per-frame register FFT (default); 0: the general block-per-frame kernel of stft.cu
extern "C" int evk_set_mel_variant(int32_t v) { g_mel_variant = v ? 1 : 0; return EVK_OK; }

static int frames_of(int L, int hop) { return (L + 2 * ((NFFT - hop) / 2) - NFFT) / hop + 1; }

extern "C" int evk_mel_fwd(const float* wav, const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t hop, int32_t n_mels,
                           const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val, float* spec,
                           int32_t ld_spec, float* mel, int32_t ld_mel, float* cplx, evk_stream_t stream) {
  EVK_REQUIRE(wav && B >= 1 && hop >= 1 && hop <= NFFT, EVK_ERR_ARG, "mel_fwd: bad arguments");
  EVK_REQUIRE(L > (NFFT - hop) / 2, EVK_ERR_ARG, "mel_fwd: L=%d too short for reflect padding %d", L, (NFFT - hop) / 2);
  EVK_REQUIRE(!mel || (fb_ptr && fb_idx && fb_val), EVK_ERR_ARG, "mel_fwd: filterbank required");
  const int T = frames_of(L, hop);
  if (T <= 0) return EVK_OK;
  const long long nframes = (long long)B * T;
  if (g_mel_variant == 0 || n_mels > 143)
    return evk_stft_fwd(wav, lens, B, L, ldw, NFFT, hop, NFFT, (NFFT - hop) / 2, T, 1e-6f, cplx, spec, ld_spec, n_mels, fb_ptr, fb_idx, fb_val,
                        1e-5f, mel, ld_mel, stream);
  int rc = mel_init_tables();
  if (rc) { set_error("mel_fwd: table init failed"); return rc; }
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(mel_fwd_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MEL_TAB_SMEM + MEL_WPB * MEL_WARP_SMEM);
    attr_set = true;
  }
  const long long need = (nframes + MEL_WPB - 1) / MEL_WPB;
  const unsigned grid = (unsigned)(need < 2 * kNumSMs ? need : 2 * kNumSMs);            // persistent: two CTAs per SM
  mel_fwd_warp_kernel<<<grid, MEL_WPB * 32, MEL_TAB_SMEM + MEL_WPB * MEL_WARP_SMEM, (cudaStream_t)stream>>>(
      wav, lens, L, ldw, T, nframes, hop, n_mels, fb_ptr, fb_idx, fb_val, spec, ld_spec, mel, ld_mel, cplx);
  return check_launch("mel_fwd_warp_kernel");
}

// adjoint of the log-mel front end (loss_mel): one more forward FFT per frame in the general kernel (stft.cu)
extern "C" int evk_mel_bwd(const float* dmel, int32_t ld_dmel, const float* cplx, const float* mel, int32_t ld_mel,
                           const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t hop, int32_t n_mels, const int32_t* fb_ptr,
                           const int32_t* fb_idx, const float* fb_val, float* dwav, evk_stream_t stream) {
  EVK_REQUIRE(dmel && cplx && mel && dwav && fb_ptr && fb_idx && fb_val, EVK_ERR_ARG, "mel_bwd: null tensor");
  const int T = frames_of(L, hop);
  if (T <= 0) return EVK_OK;
  return evk_stft_bwd(nullptr, dmel, ld_dmel, cplx, mel, ld_mel, 1e-6f, 1e-5f, n_mels, fb_ptr, fb_idx, fb_val, lens, B, L, ldw, NFFT, hop, NFFT,
                      (NFFT - hop) / 2, T, dwav, stream);
}

extern "C" int evk_spec_to_mel(const float* spec, int64_t rows, int32_t ld_spec, int32_t n_mels, const int32_t* fb_ptr,
                               const int32_t* fb_idx, const float* fb_val, float* mel, int32_t ld_mel,
                               evk_stream_t stream) {
  EVK_REQUIRE(spec && mel && fb_ptr && fb_idx && fb_val, EVK_ERR_ARG, "spec_to_mel: null tensor");
  if (rows <= 0) return EVK_OK;
  spec_to_mel_kernel<<<(unsigned)rows, 128, 0, (cudaStream_t)stream>>>(spec, rows, ld_spec, n_mels, fb_ptr, fb_idx,
                                                                       fb_val, mel, ld_mel);
  return check_launch("spec_to_mel_kernel");
}
