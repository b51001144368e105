// General STFT front end and its adjoint (runtime n_fft = 256 .. 4096, hop, win <= n_fft, any reflect padding, per-row
// lengths): complex spectrum, |X| and log-mel of every frame, one thread block per frame, fp32 Stockham FFT in shared memory
// (index arithmetic in stft_core.cuh, validated on the host against numpy by tests/test_cpu_stft_core.py).
//   forward : spectrogram_torch / spec_to_mel_torch / mel_spectrogram_torch of mel_processing.py:40-142 for any
//             (n_fft, hop, win), and torch.stft(center=True, return_complex=True) of bs_roformer.py:565-581 (MR-STFT loss)
//   backward: d wav from d log-mel (loss_mel, sovits.py:513) or from a complex spectrum gradient (MR-STFT), through ONE
//             more forward FFT per frame (the O(N^2) inverse DFT of round 1 is gone)
// The 2048-point, center=False, log-mel / |X| fast path stays in mel.cu (warp-per-frame register FFT).
#include "evk_common.cuh"
#include <math.h>

#include "stft_core.cuh"

namespace evk {

__device__ float2 g_stw[STFT_TAB];      // e^{-2 pi i k / 4096}
__device__ float g_shann[STFT_TAB];     // periodic Hann(4096)
static bool g_stft_ready = false;

int stft_init_tables() {
  if (g_stft_ready) return EVK_OK;
  static float2 tw[STFT_TAB];
  static float hw[STFT_TAB];
  for (int i = 0; i < STFT_TAB; ++i) {
    const double a = 2.0 * M_PI * (double)i / (double)STFT_TAB;
    tw[i] = make_float2((float)cos(a), (float)(-sin(a)));
    hw[i] = (float)(0.5 - 0.5 * cos(a));
  }
  if (cudaMemcpyToSymbol(g_stw, tw, sizeof(tw)) != cudaSuccess) return EVK_ERR_CUDA;
  if (cudaMemcpyToSymbol(g_shann, hw, sizeof(hw)) != cudaSuccess) return EVK_ERR_CUDA;
  g_stft_ready = true;
  return EVK_OK;
}

namespace {

constexpr int ST_THREADS = 256;

struct StftP {
  const float* wav; const int* lens; float* dwav;
  int B, L, ldw, N, hop, win, pad, T;
  float mag_eps, clip;
  float* cplx; float* spec; int ld_spec; float* mel; int ld_mel;
  int n_mels; const int* fb_ptr; const int* fb_idx; const float* fb_val;
  // backward inputs
  const float* gcplx; const float* dmel; int ld_dmel; const float* mel_in; const float* cplx_in;
  float* frbuf;              // backward: windowed adjoint of every frame [B*T][N], overlap-added by stft_ola_kernel
};

__device__ __forceinline__ int frames_of_row(int Lrow, int pad, int N, int hop) {
  const int span = Lrow + 2 * pad - N;
  return span < 0 ? 0 : span / hop + 1;
}

// shared memory: d0[NH] d1[NH] float2 | sx[NH + 1] float2 | mag[NH + 1 (+3)] float
__device__ __forceinline__ const float2* run_fft(int NH, float2* d0, float2* d1) {
  float2 *src = d0, *dst = d1;
  for (int Ns = 1; Ns < NH;) {
    Ns = stft_pass(threadIdx.x, ST_THREADS, NH, Ns, src, dst, g_stw);
    __syncthreads();
    float2* t = src; src = dst; dst = t;
  }
  return src;
}

__global__ void __launch_bounds__(ST_THREADS) stft_fwd_kernel(const StftP p) {
  extern __shared__ __align__(16) uint8_t ssm[];
  const int NH = p.N >> 1, NB = NH + 1;
  float2* d0 = reinterpret_cast<float2*>(ssm);
  float2* d1 = d0 + NH;
  float2* sx = d1 + NH;
  float* mag = reinterpret_cast<float*>(sx + NB + 1);
  const long long frame = blockIdx.x;
  const int b = (int)(frame / p.T), f = (int)(frame - (long long)b * p.T);
  const int Lrow = p.lens ? min(p.lens[b], p.L) : p.L;
  const int tid = threadIdx.x;
  if (f >= frames_of_row(Lrow, p.pad, p.N, p.hop)) {         // past this row's own last frame: what the zero-padded collate holds
    for (int k = tid; k < NB; k += ST_THREADS) {
      if (p.spec) p.spec[frame * p.ld_spec + k] = 0.f;
      if (p.cplx) reinterpret_cast<float2*>(p.cplx)[frame * NB + k] = make_float2(0.f, 0.f);
    }
    if (p.mel)
      for (int m = tid; m < p.n_mels; m += ST_THREADS) p.mel[frame * p.ld_mel + m] = logf(p.clip);
    return;
  }
  stft_load_phase(tid, ST_THREADS, p.wav + (long long)b * p.ldw, Lrow, f * p.hop - p.pad, p.N, p.win, g_shann, d0);
  __syncthreads();
  const float2* z = run_fft(NH, d0, d1);
  stft_untangle_phase(tid, ST_THREADS, p.N, z, g_stw, sx);
  __syncthreads();
  for (int k = tid; k < NB; k += ST_THREADS) {
    const float2 x = sx[k];
    if (p.cplx) reinterpret_cast<float2*>(p.cplx)[frame * NB + k] = x;
    if (p.spec || p.mel) {
      const float m = sqrtf(x.x * x.x + x.y * x.y + p.mag_eps);
      mag[k] = m;
      if (p.spec) p.spec[frame * p.ld_spec + k] = m;
    }
  }
  if (p.mel) {
    __syncthreads();
    for (int m = tid; m < p.n_mels; m += ST_THREADS) {
      float acc = 0.f;
      for (int e = p.fb_ptr[m]; e < p.fb_ptr[m + 1]; ++e) acc = fmaf(p.fb_val[e], mag[p.fb_idx[e]], acc);
      p.mel[frame * p.ld_mel + m] = logf(fmaxf(acc, p.clip));
    }
  }
}

// adjoint of one frame, windowed, into frbuf; stft_ola_kernel then overlap-adds the frames into dwav through the same reflect
// indexing the forward read with (a gather in fixed frame order: reproducible, unlike atomics)
__global__ void __launch_bounds__(ST_THREADS) stft_bwd_kernel(const StftP p) {
  extern __shared__ __align__(16) uint8_t ssm[];
  const int NH = p.N >> 1, NB = NH + 1;
  float2* d0 = reinterpret_cast<float2*>(ssm);
  float2* d1 = d0 + NH;
  float2* G = d1 + NH;
  float* dmag = reinterpret_cast<float*>(G + NB + 1);
  const long long frame = blockIdx.x;
  const int b = (int)(frame / p.T), f = (int)(frame - (long long)b * p.T);
  const int Lrow = p.lens ? min(p.lens[b], p.L) : p.L;
  const int tid = threadIdx.x;
  if (f >= frames_of_row(Lrow, p.pad, p.N, p.hop)) return;    // uniform per block
  if (p.gcplx) {
    for (int k = tid; k < NB; k += ST_THREADS) G[k] = reinterpret_cast<const float2*>(p.gcplx)[frame * NB + k];
  } else {
    // d log(clamp(s, clip)) / ds = 1/s where s >= clip (torch.clamp passes the gradient at s >= min); s = exp(log-mel)
    float* gm = reinterpret_cast<float*>(d1);                   // per-mel gradient (d1 is free until the FFT)
    for (int k = tid; k < NB; k += ST_THREADS) dmag[k] = 0.f;
    const float lclip = logf(p.clip);
    for (int m = tid; m < p.n_mels; m += ST_THREADS) {
      const float lm = p.mel_in[frame * p.ld_mel + m];
      gm[m] = (lm > lclip) ? p.dmel[frame * p.ld_dmel + m] * expf(-lm) : 0.f;
    }
    __syncthreads();
    // filterbank transpose in mel order: the bins of one filter are distinct, so a bin receives its filters' terms in m order
    for (int m = 0; m < p.n_mels; ++m) {
      const float g = gm[m];
      if (g != 0.f)
        for (int e = p.fb_ptr[m] + tid; e < p.fb_ptr[m + 1]; e += ST_THREADS) dmag[p.fb_idx[e]] += p.fb_val[e] * g;
      __syncthreads();
    }
    for (int k = tid; k < NB; k += ST_THREADS) {
      const float2 x = reinterpret_cast<const float2*>(p.cplx_in)[frame * NB + k];
      const float s = dmag[k] / sqrtf(x.x * x.x + x.y * x.y + p.mag_eps);
      G[k] = make_float2(s * x.x, s * x.y);
    }
  }
  __syncthreads();
  stft_adjoint_pack_phase(tid, ST_THREADS, p.N, G, g_stw, d0);
  __syncthreads();
  const float2* r = run_fft(NH, d0, d1);
  float* fr = p.frbuf + frame * p.N;
  for (int m = tid; m < NH; m += ST_THREADS) {
    const float2 v = r[m];
    const int n0 = 2 * m, n1 = n0 + 1;
    const float w0 = stft_window(g_shann, n0, p.N, p.win), w1 = stft_window(g_shann, n1, p.N, p.win);
    fr[n0] = v.x * w0;
    fr[n1] = -v.y * w1;
  }
}

// dwav[b][n] += sum over the padded positions s that reflect onto n (s = n, -n, 2 (Lrow - 1) - n, in that order) and over
// the frames f covering s (ascending) of frbuf[b*T + f][s - f*hop + pad]
__global__ void stft_ola_kernel(const StftP p) {
  const long long total = (long long)p.B * p.L;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / p.L), n = (int)(i - (long long)b * p.L);
    const int Lrow = p.lens ? min(p.lens[b], p.L) : p.L;
    if (n >= Lrow) continue;
    const int nf = min(frames_of_row(Lrow, p.pad, p.N, p.hop), p.T);   // frbuf holds T frames per row
    const int cand[3] = {n, -n, 2 * (Lrow - 1) - n};
    float acc = 0.f;
    for (int ci = 0; ci < 3; ++ci) {
      const int s = cand[ci];
      if ((ci == 1 && n == 0) || (ci == 2 && cand[2] == n) || stft_reflect(s, Lrow) != n) continue;
      const int hi = (s + p.pad) >= 0 ? (s + p.pad) / p.hop : -1;                      // last frame starting at or before s
      int lo = s + p.pad - p.N + 1;                                                      // first frame whose span reaches s
      lo = lo <= 0 ? 0 : (lo + p.hop - 1) / p.hop;
      for (int f = lo; f <= hi && f < nf; ++f) acc += p.frbuf[((long long)b * p.T + f) * p.N + (s - f * p.hop + p.pad)];
    }
    p.dwav[(long long)b * p.ldw + n] += acc;
  }
}

// loss += scale * sum_i |a_i - b_i| over complex elements (F.l1_loss on complex tensors = mean modulus of the difference),
// g_i = scale * (a_i - b_i) / |a_i - b_i|   (gradient wrt a as (d/dRe, d/dIm); 0 where a == b)
__global__ void __launch_bounds__(256) cplx_l1_kernel(const float2* __restrict__ a, const float2* __restrict__ b, long long n, float scale,
                                                      float* __restrict__ loss, float2* __restrict__ grad) {
  __shared__ float red[33];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float2 x = a[i], y = b[i];
    const float dx = x.x - y.x, dy = x.y - y.y;
    const float m = sqrtf(dx * dx + dy * dy);
    acc += m;
    if (grad) {
      const float inv = m > 0.f ? scale / m : 0.f;
      grad[i] = make_float2(dx * inv, dy * inv);
    }
  }
  const float tot = block_sum(acc, red);
  if (threadIdx.x == 0) loss[blockIdx.x] = tot * scale;      // per-block partial (ordered_sum adds them)
}

// Inverse STFT (torch.istft(center=True, normalized=False, onesided, length=None) with the Hann(n_fft) window), optionally of
// stft * mask (bs_roformer.py:530-543): one block per frame (row r = b S + s, frame t) runs the C2R inverse DFT through the same
// adjoint packing and forward FFT as stft_bwd_kernel (bins 0 and N/2 lose their imaginary parts), windows the frame and writes it
// to work [(r T + t)][N]; istft_ola_kernel then overlap-adds the frames in frame order and divides by the sum of w^2.
struct IstftP {
  const float2* cplx; const float* mask; int ldm;
  int S, T, N, hop;
  float* work; float* out; int ldo; int Lout;
};

__global__ void __launch_bounds__(ST_THREADS) istft_frame_kernel(const IstftP p) {
  extern __shared__ __align__(16) uint8_t ssm[];
  const int NH = p.N >> 1, NB = NH + 1;
  float2* d0 = reinterpret_cast<float2*>(ssm);
  float2* d1 = d0 + NH;
  float2* G = d1 + NH;
  const long long frame = blockIdx.x;
  const int r = (int)(frame / p.T), t = (int)(frame - (long long)r * p.T);
  const int b = r / p.S, s = r - b * p.S;
  const int tid = threadIdx.x;
  const float inv = 1.f / (float)p.N;
  for (int k = tid; k < NB; k += ST_THREADS) {
    float2 x = p.cplx[frame * NB + k];
    if (p.mask) {           // mask row (b, t), column ((k S + s), c): the mask estimator's 'b t (f s c)' layout
      const float2 m = *reinterpret_cast<const float2*>(p.mask + ((long long)b * p.T + t) * p.ldm + 2 * (k * p.S + s));
      x = stft_cmul(x, m);
    }
    const float sc = (k == 0 || k == NH) ? inv : 2.f * inv;  // irfft(X)[n] = sum_k Re(G[k] e^{2 pi i k n / N}) with these weights
    G[k] = make_float2(x.x * sc, x.y * sc);
  }
  __syncthreads();
  stft_adjoint_pack_phase(tid, ST_THREADS, p.N, G, g_stw, d0);
  __syncthreads();
  const float2* z = run_fft(NH, d0, d1);
  float* fr = p.work + frame * p.N;
  for (int m = tid; m < NH; m += ST_THREADS) {
    const float2 v = z[m];
    fr[2 * m] = v.x * stft_window(g_shann, 2 * m, p.N, p.N);
    fr[2 * m + 1] = -v.y * stft_window(g_shann, 2 * m + 1, p.N, p.N);
  }
}

// out[r][n] = sum_f frame_f[q - f hop] / sum_f w(q - f hop)^2 over the frames covering q = n + N/2 (ascending f)
__global__ void istft_ola_kernel(const IstftP p) {
  const int r = blockIdx.y;
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < p.Lout; n += (long long)gridDim.x * blockDim.x) {
    const int q = (int)n + (p.N >> 1);
    int lo = q - p.N + 1;
    lo = lo <= 0 ? 0 : (lo + p.hop - 1) / p.hop;
    const int hi = min(q / p.hop, p.T - 1);
    float y = 0.f, env = 0.f;
    for (int f = lo; f <= hi; ++f) {
      const int j = q - f * p.hop;
      const float w = stft_window(g_shann, j, p.N, p.N);
      y += p.work[((long long)r * p.T + f) * p.N + j];
      env += w * w;
    }
    p.out[(long long)r * p.ldo + n] = y / env;
  }
}

int fill(StftP& p, const float* wav, const int32_t* lens, int B, int L, int ldw, int n_fft, int hop, int win, int pad, int T) {
  EVK_REQUIRE(B > 0 && L > 0 && T > 0 && hop > 0 && pad >= 0 && ldw >= L, EVK_ERR_ARG, "stft: bad sizes B=%d L=%d T=%d hop=%d pad=%d", B, L, T, hop, pad);
  EVK_REQUIRE(n_fft >= 256 && n_fft <= STFT_TAB && (n_fft & (n_fft - 1)) == 0, EVK_ERR_UNSUPPORTED, "stft: n_fft=%d must be a power of two in [256, 4096]", n_fft);
  EVK_REQUIRE(win >= 2 && win <= n_fft && (win & (win - 1)) == 0, EVK_ERR_UNSUPPORTED, "stft: win=%d must be a power of two <= n_fft", win);
  EVK_REQUIRE(pad < L, EVK_ERR_ARG, "stft: reflect padding %d must be smaller than the signal length %d", pad, L);
  EVK_REQUIRE((long long)(T - 1) * hop - pad + n_fft <= (long long)L + pad, EVK_ERR_ARG, "stft: T=%d frames do not fit L=%d with padding %d", T, L, pad);
  p.wav = wav; p.lens = lens; p.B = B; p.L = L; p.ldw = ldw; p.N = n_fft; p.hop = hop; p.win = win; p.pad = pad; p.T = T;
  return stft_init_tables();
}

size_t smem_for(int n_fft) { return (size_t)(n_fft / 2) * 16 + (size_t)(n_fft / 2 + 2) * 8 + (size_t)(n_fft / 2 + 4) * 4; }

template <typename K>
int launch(K kern, const StftP& p, cudaStream_t st, const char* name) {
  const size_t smem = smem_for(p.N);
  static size_t attr_fwd = 0, attr_bwd = 0;
  size_t& cur = (reinterpret_cast<const void*>(kern) == reinterpret_cast<const void*>(stft_fwd_kernel)) ? attr_fwd : attr_bwd;
  if (smem > cur) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return check_launch(name);
    cur = smem;
  }
  const long long frames = (long long)p.B * p.T;
  EVK_REQUIRE(frames <= 0x7fffffff, EVK_ERR_ARG, "%s: too many frames", name);
  kern<<<(unsigned)frames, ST_THREADS, smem, st>>>(p);
  return check_launch(name);
}

}  // namespace
}  // namespace evk

using namespace evk;

// Frames f = 0 .. T-1 of row b start at sample f*hop - pad of the row reflect-padded by `pad` on both sides
//   mel_processing.py:40-74  : pad = (n_fft - hop) / 2, T = (L + 2 pad - n_fft) / hop + 1   (center=False after a manual pad)
//   torch.stft(center=True)  : pad = n_fft / 2,         T = 1 + L / hop
// lens (nullable, int32 [B]): per-row valid length -- the reflection then sits at each row's OWN end and frames past the
// row's own count are written as the zero-padded collate holds them (|X| = 0, log-mel = log(clip)).
// Outputs (each nullable): cplx [B*T][n_fft/2+1][2], spec [B*T][ld_spec] = sqrt(re^2 + im^2 + mag_eps),
// mel [B*T][ld_mel] = log(max(filterbank . spec, clip)) with the filterbank in CSR-by-mel form.
extern "C" int evk_stft_fwd(const float* wav, const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t n_fft, int32_t hop, int32_t win,
                            int32_t pad, int32_t T, float mag_eps, float* cplx, float* spec, int32_t ld_spec, int32_t n_mels,
                            const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val, float clip, float* mel, int32_t ld_mel,
                            evk_stream_t stream) {
  StftP p{};
  int rc = fill(p, wav, lens, B, L, ldw, n_fft, hop, win, pad, T);
  if (rc) return rc;
  EVK_REQUIRE(wav && (cplx || spec || mel), EVK_ERR_ARG, "stft_fwd: null input or no output requested");
  EVK_REQUIRE(!mel || (fb_ptr && fb_idx && fb_val && n_mels > 0 && ld_mel >= n_mels), EVK_ERR_ARG, "stft_fwd: mel output needs a filterbank");
  EVK_REQUIRE(!spec || ld_spec >= n_fft / 2 + 1, EVK_ERR_ARG, "stft_fwd: ld_spec too small");
  p.mag_eps = mag_eps; p.clip = clip; p.cplx = cplx; p.spec = spec; p.ld_spec = ld_spec; p.mel = mel; p.ld_mel = ld_mel;
  p.n_mels = n_mels; p.fb_ptr = fb_ptr; p.fb_idx = fb_idx; p.fb_val = fb_val;
  return launch(stft_fwd_kernel, p, (cudaStream_t)stream, "stft_fwd_kernel");
}

// dwav [B][ldw] += adjoint.  Either gcplx [B*T][n_fft/2+1][2] (dL/dRe, dL/dIm of the complex spectrum) or the log-mel path:
// dmel [B*T][ld_dmel] with the forward's saved cplx and mel.  dwav must be zero-initialised by the caller (overlap-add).
extern "C" int evk_stft_bwd(const float* gcplx, const float* dmel, int32_t ld_dmel, const float* cplx, const float* mel, int32_t ld_mel,
                            float mag_eps, float clip, int32_t n_mels, const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val,
                            const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t n_fft, int32_t hop, int32_t win, int32_t pad,
                            int32_t T, float* dwav, evk_stream_t stream) {
  StftP p{};
  int rc = fill(p, dwav, lens, B, L, ldw, n_fft, hop, win, pad, T);
  if (rc) return rc;
  EVK_REQUIRE(dwav && (gcplx || (dmel && cplx && mel && fb_ptr && fb_idx && fb_val && n_mels > 0)), EVK_ERR_ARG, "stft_bwd: missing gradient inputs");
  p.dwav = dwav; p.gcplx = gcplx; p.dmel = dmel; p.ld_dmel = ld_dmel; p.cplx_in = cplx; p.mel_in = mel; p.ld_mel = ld_mel;
  p.mag_eps = mag_eps; p.clip = clip; p.n_mels = n_mels; p.fb_ptr = fb_ptr; p.fb_idx = fb_idx; p.fb_val = fb_val;
  EVK_REQUIRE(gcplx || n_mels <= n_fft, EVK_ERR_ARG, "stft_bwd: n_mels > n_fft");
  Scratch fr_buf((long long)B * T * n_fft, (cudaStream_t)stream);
  p.frbuf = fr_buf.p;
  EVK_REQUIRE(p.frbuf, EVK_ERR_CUDA, "stft_bwd: scratch allocation failed");
  if (int rc2 = launch(stft_bwd_kernel, p, (cudaStream_t)stream, "stft_bwd_kernel")) return rc2;
  const long long total = (long long)B * L;
  const long long blocks = (total + 255) / 256;
  stft_ola_kernel<<<(unsigned)(blocks < kNumSMs * 16 ? blocks : kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(p);
  return check_launch("stft_ola_kernel");
}

extern "C" int evk_istft(const float* cplx, const float* mask, int32_t ld_mask, int32_t B, int32_t S, int32_t T, int32_t n_fft,
                         int32_t hop, float* work, float* out, int32_t ld_out, evk_stream_t stream) {
  EVK_REQUIRE(cplx && work && out, EVK_ERR_ARG, "istft: null tensor");
  EVK_REQUIRE(n_fft >= 256 && n_fft <= STFT_TAB && (n_fft & (n_fft - 1)) == 0, EVK_ERR_UNSUPPORTED, "istft: n_fft=%d must be a power of two in [256, 4096]", n_fft);
  EVK_REQUIRE(B > 0 && S > 0 && T >= 2 && hop > 0 && hop <= n_fft / 2 && (long long)B * S <= 65535, EVK_ERR_ARG,
              "istft: bad sizes B=%d S=%d T=%d hop=%d", B, S, T, hop);
  EVK_REQUIRE(!mask || (ld_mask >= 2 * S * (n_fft / 2 + 1) && (uintptr_t)mask % 8 == 0 && ld_mask % 2 == 0), EVK_ERR_ARG,
              "istft: mask rows must hold 2 * S * (n_fft / 2 + 1) floats, 8-byte aligned");
  const long long Lout = (long long)hop * (T - 1), frames = (long long)B * S * T;
  EVK_REQUIRE(ld_out >= Lout && frames <= 0x7fffffff && Lout <= 0x7fffffff, EVK_ERR_ARG, "istft: output pitch %d < %lld", ld_out, Lout);
  if (int rc = stft_init_tables()) return rc;
  IstftP p{reinterpret_cast<const float2*>(cplx), mask, ld_mask, S, T, n_fft, hop, work, out, ld_out, (int)Lout};
  const size_t smem = (size_t)(n_fft / 2) * 16 + (size_t)(n_fft / 2 + 1) * 8;
  static size_t attr = 48 * 1024;
  if (smem > attr) {
    if (cudaFuncSetAttribute(istft_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return check_launch("istft_frame_kernel");
    attr = smem;
  }
  cudaStream_t st = (cudaStream_t)stream;
  istft_frame_kernel<<<(unsigned)frames, ST_THREADS, smem, st>>>(p);
  if (int rc = check_launch("istft_frame_kernel")) return rc;
  const long long bx = (Lout + 255) / 256;
  istft_ola_kernel<<<dim3((unsigned)(bx < 1024 ? bx : 1024), (unsigned)(B * S)), 256, 0, st>>>(p);
  return check_launch("istft_ola_kernel");
}

// loss[0] += scale * sum |a - b| over n complex elements; grad (nullable) = scale * (a - b) / |a - b|
extern "C" int evk_cplx_l1(const float* a, const float* b, int64_t n, float scale, float* loss, float* grad, evk_stream_t stream) {
  EVK_REQUIRE(a && b && loss && n > 0, EVK_ERR_ARG, "cplx_l1: null argument");
  const int blocks = (int)min((long long)kNumSMs * 8, (long long)((n + 255) / 256));
  Scratch part_buf(blocks, (cudaStream_t)stream);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "cplx_l1: scratch allocation failed");
  cplx_l1_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(a), reinterpret_cast<const float2*>(b), n, scale, part,
                                                          reinterpret_cast<float2*>(grad));
  if (int rc = check_launch("cplx_l1_kernel")) return rc;
  return ordered_sum(part, blocks, 1, 1, 1, loss, 0, 0, (cudaStream_t)stream);
}
