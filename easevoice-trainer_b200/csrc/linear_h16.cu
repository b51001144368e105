// 16-bit Linears (sm_90a):  y[r][n] = act( sum_k h(x[r][k]) * w[n][k] + bias[n] + res[r][n] )
// h = round to nearest even to fp16 or bf16 (cvt.rn), applied to the fp32 activations as they are staged; w is already
// 16-bit (ops.pack_weight_h16).  Products of two 16-bit values are exact in fp32 and accumulate in fp32 on the tensor
// cores; the epilogue is fp32.  The numerical contract is in include/evk.h.
//
//   evk_linear_rows_h16  the decode step's few rows: mma.sync.m16n8k16.  A CTA owns 64 output columns (8 warps x 8) and a
//                        K range whose size depends on (N, K) only; it stages the rows' activations in 64-wide K chunks
//                        as 16 bits in shared memory (shared by its 8 warps) and streams its weight slice from HBM once
//                        per 128 rows.  K splits store fp32 partials that one pass adds in split order.
//   evk_linear_h16       many rows (the encoder, the cross K/V projection): the fp32 input is cast to 16 bits in library
//                        scratch, then a TMA-fed wgmma.m64n128k16 kernel in the style of gemm_tma.cu (one producer warp, two
//                        consumer warpgroups of 64 rows, 128-byte swizzle, a ring of 5 stages of 64 K), no K split.
#include <algorithm>

#include "wgmma.cuh"

namespace evk {
namespace {

__device__ __forceinline__ float epi(float acc, const float* bias, const float* res, size_t ridx, int n, int act, float slope) {
  float v = acc;
  if (bias) v += bias[n];
  if (res) v += res[ridx];
  return conv_act(v, act, slope);
}

// ---- row kernel ---------------------------------------------------------------------------------------------------------
constexpr int RK_WARPS = 8, RK_THREADS = 32 * RK_WARPS, RK_BN = 8 * RK_WARPS, RK_RB = 128, RK_KC = 64;
constexpr int RK_STAGE = RK_RB * RK_KC / RK_THREADS;          // activations a thread stages per chunk

struct RowsP {
  const float* x; int ldx, rows;
  const uint16_t* w; int ldw;
  const float* bias; const float* res; int ldr;
  float* y; int ldy;
  int N, K, act; float slope;
  int chunks_per_split, splits;
  float* part;                                                 // splits > 1: [splits][rows][N] partials
};

// Lane (g, t) of warp v holds the weight fragment w[n0 + 8v + g][64c + 8t .. + 7] and [64c + 32 + 8t .. + 7] of chunk c (two
// 16-byte loads; 4 lanes read 64 contiguous bytes of a weight row).  K is permuted inside each 16-wide MMA step -- logical
// k slots 2t, 2t+1 hold physical 8t, 8t+1 and slots 2t+8, 2t+9 hold 8t+2, 8t+3 (then 8t+4.. and 8t+6.. in the second step) --
// and the A fragments follow the same permutation, so the contraction is unchanged.  The staged activations are [128][32]
// 16-bit per half chunk: a lane's 16-byte read of row g at 16 t is conflict-free.
template <bool BF16>
__global__ void __launch_bounds__(RK_THREADS) linear_rows_h16_kernel(const RowsP p) {
  __shared__ __align__(16) uint16_t xs[2][2][RK_RB * 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int n_w = blockIdx.x * RK_BN + warp * 8;
  const int nk = (p.K + RK_KC - 1) / RK_KC;
  const int c0 = blockIdx.y * p.chunks_per_split, c1 = min(nk, c0 + p.chunks_per_split);
  const bool w_ok = n_w + g < p.N;
  const uint16_t* wrow = p.w + (size_t)(w_ok ? n_w + g : 0) * p.ldw + 8 * t;

  for (int r0 = 0; r0 < p.rows; r0 += RK_RB) {
    const int nr = min(RK_RB, p.rows - r0), mts = (nr + 15) >> 4, nst = mts * 16 * RK_KC;
    float acc[RK_RB / 16][4];
#pragma unroll
    for (int i = 0; i < RK_RB / 16; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    float xr[RK_STAGE];
    uint4 wc0, wc1, wn0, wn1;
    // element e of a chunk: row e / 64, k = e % 64 (a warp reads 32 consecutive k of one row); half = k / 32
    auto load_x = [&](int c) {
#pragma unroll
      for (int i = 0; i < RK_STAGE; ++i) {
        const int e = tid + RK_THREADS * i, r = e >> 6, k = c * RK_KC + (e & 63);
        xr[i] = (e < nst && r < nr && k < p.K) ? __ldg(p.x + (size_t)(r0 + r) * p.ldx + k) : 0.f;
      }
    };
    auto store_x = [&](int buf) {
#pragma unroll
      for (int i = 0; i < RK_STAGE; ++i) {
        const int e = tid + RK_THREADS * i;
        if (e < nst) xs[buf][(e >> 5) & 1][(e >> 6) * 32 + (e & 31)] = to_h16<BF16>(xr[i]);
      }
    };
    auto load_w = [&](int c, uint4& a, uint4& b) {
      if (w_ok) {
        a = __ldg(reinterpret_cast<const uint4*>(wrow + c * RK_KC));
        b = __ldg(reinterpret_cast<const uint4*>(wrow + c * RK_KC + 32));
      } else {
        a = b = make_uint4(0u, 0u, 0u, 0u);
      }
    };
    __syncthreads();                                           // the previous row block's last chunk is read
    if (c0 < c1) {
      load_x(c0);
      load_w(c0, wc0, wc1);
      store_x(0);
    }
    for (int c = c0; c < c1; ++c) {
      const int buf = (c - c0) & 1;
      __syncthreads();
      const bool more = c + 1 < c1;
      if (more) {
        load_x(c + 1);
        load_w(c + 1, wn0, wn1);
      }
#pragma unroll
      for (int mt = 0; mt < RK_RB / 16; ++mt) {
        if (mt < mts) {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const uint4 lo = *reinterpret_cast<const uint4*>(&xs[buf][hf][(mt * 16 + g) * 32 + 8 * t]);
            const uint4 hi = *reinterpret_cast<const uint4*>(&xs[buf][hf][(mt * 16 + g + 8) * 32 + 8 * t]);
            const uint4 wv = hf ? wc1 : wc0;
            mma16816<BF16>(acc[mt], lo.x, hi.x, lo.y, hi.y, wv.x, wv.y);
            mma16816<BF16>(acc[mt], lo.z, hi.z, lo.w, hi.w, wv.z, wv.w);
          }
        }
      }
      if (more) {
        store_x(buf ^ 1);
        wc0 = wn0;
        wc1 = wn1;
      }
    }
#pragma unroll
    for (int mt = 0; mt < RK_RB / 16; ++mt) {
      if (mt >= mts) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = mt * 16 + g + 8 * h;
        if (r >= nr) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n_w + 2 * t + e;
          if (n >= p.N) continue;
          const float v = acc[mt][2 * h + e];
          if (p.splits == 1) p.y[(size_t)(r0 + r) * p.ldy + n] = epi(v, p.bias, p.res, (size_t)(r0 + r) * p.ldr + n, n, p.act, p.slope);
          else p.part[((size_t)blockIdx.y * p.rows + r0 + r) * p.N + n] = v;
        }
      }
    }
  }
}

// The K splits' partials added in split order, then the epilogue.
__global__ void rows_h16_reduce_kernel(const RowsP p) {
  const long long total = (long long)p.rows * p.N, ps = total;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / p.N), n = (int)(i - (long long)r * p.N);
    float v = p.part[i];
    for (int s = 1; s < p.splits; ++s) v += p.part[s * ps + i];
    p.y[(size_t)r * p.ldy + n] = epi(v, p.bias, p.res, (size_t)r * p.ldr + n, n, p.act, p.slope);
  }
}

// ---- many-row kernel ----------------------------------------------------------------------------------------------------
constexpr int LB_M = 128, LB_N = 128, LB_K = 64, LB_STAGES = 5, LB_THREADS = 384;
constexpr int LB_A = LB_M * LB_K * 2, LB_B = LB_N * LB_K * 2, LB_STAGE = LB_A + LB_B;
constexpr int LB_SMEM = LB_STAGES * LB_STAGE + 1024;

struct LinP {
  const float* bias; const float* res; int ldr;
  float* y; int ldy;
  int M, N, K, act; float slope;
};

// x [M][ldx] fp32 -> xh [M][Kc] 16-bit (Kc = K rounded up to 8; zeros past K), 8 values per thread and step.
template <bool BF16>
__global__ void cast_h16_kernel(const float* __restrict__ x, int ldx, int M, int K, int Kc, uint4* __restrict__ xh) {
  const int per_row = Kc / 8;
  const long long total = (long long)M * per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / per_row), k0 = (int)(i - (long long)r * per_row) * 8;
    const float* src = x + (size_t)r * ldx;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = k0 + e < K ? __ldg(src + k0 + e) : 0.f;
    xh[i] = make_uint4(to_h16x2<BF16>(v[0], v[1]), to_h16x2<BF16>(v[2], v[3]), to_h16x2<BF16>(v[4], v[5]), to_h16x2<BF16>(v[6], v[7]));
  }
}

template <bool BF16>
__global__ void __launch_bounds__(LB_THREADS, 1) linear_h16_kernel(const __grid_constant__ CUtensorMap mapA,
                                                                   const __grid_constant__ CUtensorMap mapB, const LinP p) {
  extern __shared__ uint8_t lsm_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(lsm_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full[LB_STAGES], empty[LB_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * LB_M, n0 = blockIdx.x * LB_N;
  const int nkb = (p.K + LB_K - 1) / LB_K;
  if (threadIdx.x == 0) {
    for (int i = 0; i < LB_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;\n");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapA)));
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapB)));
  }
  __syncthreads();
  if (warp == 0) {
    const bool leader = elect_one();
    int s = 0, ph = 1;                                         // empty barriers: the first pass over the ring passes at once
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&empty[s], ph);
      if (leader) {
        uint8_t* st = sm + (size_t)s * LB_STAGE;
        mbar_expect_tx(&full[s], LB_STAGE);
        tma_load_2d(st, &mapA, kb * LB_K, m0, &full[s]);
        tma_load_2d(st + LB_A, &mapB, kb * LB_K, n0, &full[s]);
      }
      if (++s == LB_STAGES) { s = 0; ph ^= 1; }
    }
  } else if (warp >= 4) {
    const int cw = warp - 4, wg = cw >> 2, wq = cw & 3;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const uint32_t base = smem_u32(sm);
    int s = 0, ph = 0, rel = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&full[s], ph);
      const uint32_t st = base + (uint32_t)(s * LB_STAGE);
      const uint64_t da = wg_desc_sw128(st + (uint32_t)(wg * 64 * LB_K * 2)), db = wg_desc_sw128(st + LB_A);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < LB_K / 16; ++k) wgmma_h16_n128<BF16>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), 1u);
      wgmma_commit();
      wgmma_wait<1>();                                         // the group before this one has retired: release its stage
      if (lane == 0 && rel >= 0) mbar_arrive(&empty[rel]);
      rel = s;
      if (++s == LB_STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    // d[4j + 2h + e] = (row lane / 4 + 8h, column 8j + 2 (lane % 4) + e) of this warp's 16 rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (r >= p.M) continue;
#pragma unroll
      for (int j = 0; j < LB_N / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n0 + 8 * j + 2 * (lane & 3) + e;
          if (n < p.N) p.y[(size_t)r * p.ldy + n] = epi(acc[4 * j + 2 * h + e], p.bias, p.res, (size_t)r * p.ldr + n, n, p.act, p.slope);
        }
    }
  }
}

// [rows][K] 16-bit, row pitch ld elements: box [box_rows][64], 128-byte swizzle; rows and K past the tensor are zero-filled.
bool make_map_h16(CUtensorMap* m, const void* base, long long rows, long long K, long long ld, int box_rows, bool bf16) {
  EncodeFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)LB_K, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstr,
             box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int check_args(const char* who, const float* x, int ldx, int rows, const void* w, int ldw, const float* res, int ldr, const float* y,
               int ldy, int N, int K, int act) {
  EVK_REQUIRE(x && w && y, EVK_ERR_ARG, "%s: null operand", who);
  EVK_REQUIRE(rows >= 1 && N >= 1 && K >= 1, EVK_ERR_ARG, "%s: rows %d, N %d, K %d (each >= 1)", who, rows, N, K);
  EVK_REQUIRE(ldx >= K && ldy >= N && (!res || ldr >= N), EVK_ERR_ARG, "%s: ldx %d < K %d, ldy %d < N %d or ldr %d < N", who, ldx,
              K, ldy, N, ldr);
  EVK_REQUIRE(ldw >= K && ldw % 64 == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0, EVK_ERR_ARG,
              "%s: the weight must be packed [N][ldw] with ldw %% 64 == 0, ldw >= K and 16-byte alignment (ldw %d, K %d)", who,
              ldw, K);
  EVK_REQUIRE(act >= EVK_ACT_NONE && act <= EVK_ACT_GELU, EVK_ERR_ARG, "%s: act %d", who, act);
  return EVK_OK;
}

}  // namespace

// Splits of the row kernel's K range: enough CTAs for two per SM, at least 4 chunks (256 K) each.  The choice depends on
// N and K only, so a row's sum has one order whatever `rows` is.
static int rows_h16_splits(int N, int K, int& cps) {
  const int nk = (K + RK_KC - 1) / RK_KC, ctas_n = (N + RK_BN - 1) / RK_BN;
  const int s = max(1, min(nk / 4, (2 * kNumSMs + ctas_n - 1) / ctas_n));
  cps = (nk + s - 1) / s;
  return (nk + cps - 1) / cps;
}

}  // namespace evk

using namespace evk;

extern "C" int evk_linear_rows_h16(const float* x, int32_t ldx, int32_t rows, const void* w, int32_t ldw, int32_t bf16,
                                   const float* bias, const float* res, int32_t ldr, float* y, int32_t ldy, int32_t N, int32_t K,
                                   int32_t act, float slope, evk_stream_t stream) {
  int rc = check_args("linear_rows_h16", x, ldx, rows, w, ldw, res, ldr, y, ldy, N, K, act);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RowsP p{x, ldx, rows, static_cast<const uint16_t*>(w), ldw, bias, res, ldr, y, ldy, N, K, act, slope, 0, 0, nullptr};
  p.splits = rows_h16_splits(N, K, p.chunks_per_split);
  Scratch part(p.splits > 1 ? (long long)p.splits * rows * N : 0, st);
  EVK_REQUIRE(p.splits == 1 || part.p, EVK_ERR_CUDA, "linear_rows_h16: scratch allocation failed");
  p.part = part.p;
  dim3 grid((N + RK_BN - 1) / RK_BN, p.splits);
  if (bf16) linear_rows_h16_kernel<true><<<grid, RK_THREADS, 0, st>>>(p);
  else linear_rows_h16_kernel<false><<<grid, RK_THREADS, 0, st>>>(p);
  if (p.splits > 1) {
    const long long n = (long long)rows * N;
    rows_h16_reduce_kernel<<<(int)std::min<long long>((n + 255) / 256, 4 * kNumSMs), 256, 0, st>>>(p);
  }
  return check_launch("linear_rows_h16");
}

extern "C" int evk_linear_h16(const float* x, int32_t ldx, int32_t rows, const void* w, int32_t ldw, int32_t bf16, const float* bias,
                              const float* res, int32_t ldr, float* y, int32_t ldy, int32_t N, int32_t K, int32_t act, float slope,
                              evk_stream_t stream) {
  int rc = check_args("linear_h16", x, ldx, rows, w, ldw, res, ldr, y, ldy, N, K, act);
  if (rc) return rc;
  EVK_REQUIRE((rows + LB_M - 1) / LB_M <= 65535, EVK_ERR_ARG, "linear_h16: %d rows (at most %d)", rows, 65535 * LB_M);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int Kc = (K + 7) / 8 * 8;
  Scratch xh((long long)rows * Kc / 2, st);
  EVK_REQUIRE(xh.p, EVK_ERR_CUDA, "linear_h16: scratch allocation failed");
  CUtensorMap ma, mb;
  EVK_REQUIRE(make_map_h16(&ma, xh.p, rows, K, Kc, LB_M, bf16) && make_map_h16(&mb, w, N, K, ldw, LB_N, bf16),
              EVK_ERR_UNSUPPORTED, "linear_h16: cuTensorMapEncodeTiled unavailable or rejected the operand");
  const long long groups = (long long)rows * (Kc / 8);
  const int cgrid = (int)std::min<long long>((groups + 255) / 256, 8 * kNumSMs);
  auto kern = bf16 ? linear_h16_kernel<true> : linear_h16_kernel<false>;
  EVK_REQUIRE(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LB_SMEM) == cudaSuccess, EVK_ERR_CUDA,
              "linear_h16: shared-memory opt-in failed");
  LinP p{bias, res, ldr, y, ldy, rows, N, K, act, slope};
  dim3 grid((N + LB_N - 1) / LB_N, (rows + LB_M - 1) / LB_M);
  if (bf16) cast_h16_kernel<true><<<cgrid, 256, 0, st>>>(x, ldx, rows, K, Kc, reinterpret_cast<uint4*>(xh.p));
  else cast_h16_kernel<false><<<cgrid, 256, 0, st>>>(x, ldx, rows, K, Kc, reinterpret_cast<uint4*>(xh.p));
  kern<<<grid, LB_THREADS, LB_SMEM, st>>>(ma, mb, p);
  return check_launch("linear_h16");
}
