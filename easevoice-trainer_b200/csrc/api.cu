// Library bookkeeping: init / error reporting.
#include "evk_common.cuh"
#include <stdarg.h>

namespace evk {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return EVK_ERR_CUDA;
  }
  return EVK_OK;
}
int mel_init_tables();
double g_disp_flops[EVK_DISPATCH_SLOTS] = {0};

static cudaMemPool_t g_pool = nullptr;
void Scratch::alloc(long long n) {
  if (p) { cudaFreeAsync(p, st); p = nullptr; }
  if (n <= 0 || !g_pool) return;
  void* q = nullptr;
  if (cudaMallocFromPoolAsync(&q, (size_t)n * sizeof(float), g_pool, st) == cudaSuccess) p = static_cast<float*>(q);
  else cudaGetLastError();
}
Scratch::~Scratch() {
  if (p) cudaFreeAsync(p, st);
}

// block (32, OS_LANES) per 32 consecutive output elements: lane ty sums the partials s = ty, ty + OS_LANES, ... (its fixed share),
// then the OS_LANES sums are added in ty order -- the same order on every run, independent of scheduling
constexpr int OS_LANES = 16;
__global__ void ordered_sum_kernel(const float* __restrict__ part, int S, long long ps, int O, int R, int Cn, float* __restrict__ dst,
                                   long long d_so, long long d_sr) {
  __shared__ float red[OS_LANES][33];
  const long long n = (long long)O * R * Cn;
  for (long long i0 = (long long)blockIdx.x * 32; i0 < n; i0 += (long long)gridDim.x * 32) {
    const long long i = i0 + threadIdx.x;
    float acc = 0.f;
    if (i < n)
      for (int s = threadIdx.y; s < S; s += OS_LANES) acc += part[s * ps + i];
    red[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && i < n) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < OS_LANES; ++k) t += red[k][threadIdx.x];
      const int c = (int)(i % Cn);
      const long long orr = i / Cn;
      const int r = (int)(orr % R), o = (int)(orr / R);
      dst[o * d_so + r * d_sr + c] += t;
    }
    __syncthreads();
  }
}

int ordered_sum(const float* part, int S, long long ps, int O, int R, int Cn, float* dst, long long d_so, long long d_sr, cudaStream_t st) {
  const long long n = (long long)O * R * Cn;
  if (n <= 0) return EVK_OK;
  const long long blocks = (n + 31) / 32;
  ordered_sum_kernel<<<(unsigned)(blocks < kNumSMs * 16 ? blocks : kNumSMs * 16), dim3(32, OS_LANES), 0, st>>>(part, S, ps, O, R, Cn, dst,
                                                                                                               d_so, d_sr);
  return check_launch("ordered_sum");
}
}  // namespace evk
using namespace evk;

extern "C" const char* evk_last_error(void) { return g_err; }
extern "C" int evk_version(void) { return 100; }
extern "C" int evk_gconv_desc_size(void) { return (int)sizeof(evk_gconv_desc); }

extern "C" int evk_init(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { set_error("evk_init: no CUDA device (%s) -- there is no CPU fallback", cudaGetErrorString(e)); return EVK_ERR_CUDA; }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) { set_error("evk_init: %s", cudaGetErrorString(e)); return EVK_ERR_CUDA; }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("evk_init: device '%s' is sm_%d%d; libevk_sm90 is built for sm_90a (H100) only", prop.name, prop.major, prop.minor);
    return EVK_ERR_ARCH;
  }
  if (!g_pool) {                                   // scratch pool: keeps what it has reserved instead of returning it at every sync
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    uint64_t keep = UINT64_MAX;
    if (cudaMemPoolCreate(&g_pool, &props) != cudaSuccess ||
        cudaMemPoolSetAttribute(g_pool, cudaMemPoolAttrReleaseThreshold, &keep) != cudaSuccess) {
      g_pool = nullptr;
      set_error("evk_init: scratch memory pool creation failed");
      return EVK_ERR_CUDA;
    }
  }
  int rc = mel_init_tables();
  if (rc) { set_error("evk_init: twiddle/window table upload failed"); return rc; }
  return EVK_OK;
}

extern "C" int evk_sync_check(evk_stream_t stream) {
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("evk_sync_check: %s", cudaGetErrorString(e)); return EVK_ERR_CUDA; }
  return EVK_OK;
}

// Host-side dispatch accounting (parity tests / bench.py): algorithmic flops of every contraction launch since the last
// reset, by the kernel family that served it.  Counted when the launch is enqueued -- a CUDA-graph replay adds nothing,
// so callers account one eager step of the shape they replay.
extern "C" int evk_dispatch_stats(double* out, int32_t n) {
  EVK_REQUIRE(out && n >= 1, EVK_ERR_ARG, "dispatch_stats: null output");
  for (int i = 0; i < n && i < EVK_DISPATCH_SLOTS; ++i) out[i] = g_disp_flops[i];
  return EVK_OK;
}
extern "C" int evk_dispatch_stats_reset(void) {
  for (int i = 0; i < EVK_DISPATCH_SLOTS; ++i) g_disp_flops[i] = 0.0;
  return EVK_OK;
}
