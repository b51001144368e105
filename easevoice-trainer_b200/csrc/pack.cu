// Weight-norm + TF32 rounding + operand packing of every conv / Linear / ConvTranspose weight, and its backward.
//   forward : pa[q][d0][d1] = pb[q][d1][d0] = tf32_rn( v[d0][d1][q] * (g ? g[d0] / |v[d0]| : 1) )
//   backward: dv, dg from dpa (the tensor-core weight-gradient kernels accumulate into dpa)
// One block per output-channel row d0.  A launch packs either one weight (the job is passed by value, grid = D0) or a whole
// network: the host builds, once per network, a device table of jobs (pointers into the flat parameter arena, the packed
// arena and the packed-gradient arena are all static) and job_of_row maps each block to its job.  Packing layer by layer
// would cost 342 + 304 launches of 2-20 us per stage-2 step; the table makes that one launch each way.
// round_tf32: weights are rounded to TF32 (round-to-nearest) here, once, so the tensor-core kernels can stage them with
// cp.async and still get rounded (not truncated) operands.
#include "evk_common.cuh"

namespace evk {

extern int g_precise;

// this block's job: its table entry when there is a table, else the single job (row0 = 0)
__device__ __forceinline__ evk_pack_job row_job(const evk_pack_job& one, const evk_pack_job* jobs, const int* job_of_row) {
  return jobs ? jobs[job_of_row[blockIdx.x]] : one;
}

__global__ void __launch_bounds__(256) pack_kernel(const __grid_constant__ evk_pack_job one, const evk_pack_job* __restrict__ jobs,
                                                   const int* __restrict__ job_of_row, int round_tf32) {
  __shared__ float red[33];
  const evk_pack_job j = row_job(one, jobs, job_of_row);
  const int d0 = blockIdx.x - j.row0;
  const long long n = (long long)j.D1 * j.Q;
  const float* vr = j.v + (long long)d0 * n;
  float scale = 1.f;
  if (j.g) {
    float s = 0.f;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) s += vr[i] * vr[i];
    s = block_sum(s, red);
    scale = j.g[d0] / sqrtf(s);
  }
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const int d1 = (int)(i / j.Q), q = (int)(i - (long long)d1 * j.Q);
    float w = vr[i] * scale;
    if (round_tf32) w = __uint_as_float(f2tf32(w));
    j.pa[((long long)q * j.D0p + d0) * j.lda + d1] = w;
    if (j.pb) j.pb[((long long)q * j.D1p + d1) * j.ldb + d0] = w;
  }
}

__global__ void __launch_bounds__(256) pack_bwd_kernel(const __grid_constant__ evk_pack_job one, const evk_pack_job* __restrict__ jobs,
                                                       const int* __restrict__ job_of_row) {
  __shared__ float red[33];
  const evk_pack_job j = row_job(one, jobs, job_of_row);
  const int d0 = blockIdx.x - j.row0;
  const long long n = (long long)j.D1 * j.Q;
  const float* vr = j.v + (long long)d0 * n;
  float* dvr = j.dv + (long long)d0 * n;
  if (!j.g) {
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const int d1 = (int)(i / j.Q), q = (int)(i - (long long)d1 * j.Q);
      dvr[i] = j.dpa[((long long)q * j.D0p + d0) * j.lda + d1];
    }
    return;
  }
  float ss = 0.f, dot = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const int d1 = (int)(i / j.Q), q = (int)(i - (long long)d1 * j.Q);
    const float vv = vr[i];
    ss += vv * vv;
    dot += j.dpa[((long long)q * j.D0p + d0) * j.lda + d1] * vv;
  }
  ss = block_sum(ss, red);
  dot = block_sum(dot, red);
  const float nrm = sqrtf(ss), gg = j.g[d0];
  if (threadIdx.x == 0) j.dg[d0] = dot / nrm;
  const float sc = gg / nrm, k = dot / ss;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const int d1 = (int)(i / j.Q), q = (int)(i - (long long)d1 * j.Q);
    dvr[i] = sc * (j.dpa[((long long)q * j.D0p + d0) * j.lda + d1] - vr[i] * k);
  }
}

// Every pack entry point: `table` = jobs is a device job table with nrows rows, else jobs points to ONE job in host memory.
static int pack_launch(bool bwd, bool table, const evk_pack_job* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream) {
  const char* what = bwd ? "weight_pack_bwd" : "weight_pack";
  evk_pack_job one{};
  if (table) {
    EVK_REQUIRE(jobs && job_of_row && nrows >= 1, EVK_ERR_ARG, "%s_batched: bad arguments", what);
  } else {
    EVK_REQUIRE(jobs, EVK_ERR_ARG, "%s_one: null job", what);
    one = *jobs;
    EVK_REQUIRE(one.v && one.D0 >= 1 && one.D1 >= 1 && one.Q >= 1 && one.D0p >= one.D0 && one.lda >= one.D1 && one.row0 == 0 &&
                    (bwd ? one.dpa && one.dv && (!one.g || one.dg) : one.pa && one.D1p >= one.D1 && (!one.pb || one.ldb >= one.D0)),
                EVK_ERR_ARG, "%s_one: bad job", what);
    jobs = nullptr;
    nrows = one.D0;
  }
  if (bwd)
    pack_bwd_kernel<<<nrows, 256, 0, (cudaStream_t)stream>>>(one, jobs, job_of_row);
  else
    pack_kernel<<<nrows, 256, 0, (cudaStream_t)stream>>>(one, jobs, job_of_row, !g_precise);
  return check_launch(bwd ? "pack_bwd_kernel" : "pack_kernel");
}

}  // namespace evk
using namespace evk;

extern "C" int evk_pack_job_size(void) { return (int)sizeof(evk_pack_job); }

extern "C" int evk_weight_pack_one(const evk_pack_job* j, evk_stream_t stream) { return pack_launch(false, false, j, nullptr, 0, stream); }

extern "C" int evk_weight_pack_bwd_one(const evk_pack_job* j, evk_stream_t stream) { return pack_launch(true, false, j, nullptr, 0, stream); }

extern "C" int evk_weight_pack_batched(const evk_pack_job* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream) {
  return pack_launch(false, true, jobs, job_of_row, nrows, stream);
}

extern "C" int evk_weight_pack_bwd_batched(const evk_pack_job* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream) {
  return pack_launch(true, true, jobs, job_of_row, nrows, stream);
}
