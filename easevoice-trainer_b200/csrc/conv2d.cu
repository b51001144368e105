// 2-D convolution family of the UVR5 VR separators (CascadedASPPNet and the DeEcho / DeReverb CascadedNet, uvr5.py),
// inference only, channels-last (NHWC) fp32.
//
// A pixel (b, y, x) of an activation lives at  base + b*bs + (y*W + x)*pitch  and holds C channels from there on, so a
// layer can read or write a channel slice of a wider concat buffer (pointer advanced by the slice's channel offset).
//
//   conv2d_fwd   implicit GEMM: M = B*Ho*Wo output pixels, N = output channels, K = k*k*C (tap-major, channel-minor),
//                CTA tile 128 rows x 32 K, fp32 accumulation.  Zero padding and dilation are per axis (the DeEcho
//                net's ASPP dilates rows and columns differently).
//                Two kernels, chosen from the operands:
//                * wgmma (TF32): C, pitches and pointers allow 16-byte copies and 3xTF32 is off.  Two consumer
//                  warpgroups of 64 rows x 32 / 64 / 128 columns (the smallest that covers N), a 4-stage cp.async
//                  ring in the 128-byte-swizzle layout, operands rounded to TF32 in shared memory.
//                * mma.sync m16n8k8: everything else (the 2-channel first layer, the bridges) and 3xTF32 under
//                  evk_set_precise(1).  Eight warps of 32 x 32 over 64 columns, a 3-stage cp.async ring.
//                Kernel 1, 2 (the MDX23C 2x2 stride-2 downscale) or 3.
//                Fused epilogue: y = act(acc * scale[n] + bias[n]).  Every output is summed over K in one fixed order
//                that does not depend on the pixel's place in the launch, and there are no atomics, so a window gives
//                the same bits alone or in a batch.
//   dwconv3x3    depthwise 3x3, stride 1, zero padding = dilation (the ASPP separable branches), direct fp32.
//   resize_ac    bilinear resize with align_corners=True (Decoder's x2 upsample; an input height of 1 broadcasts).
//   mean_h       mean over the height axis (AdaptiveAvgPool2d((1, None))).
//   vr_mask_head the 1x1 output conv (no bias), sigmoid, replicate pad to out_bin rows, aggressiveness exponent,
//                x mix (NCHW) and the crop by `offset` frames on both time edges (CascadedASPPNet.predict).
#include "wgmma.cuh"

namespace evk {
namespace {

constexpr int BM = 128, BN = 64, BKC = 32, LDS = BKC + 4;   // LDS: conflict-free fragment reads (bank = 4*row + col)
constexpr int NT = 256;

struct ConvArgs {
  const float* x; const float* w; const float* scale; const float* bias; float* y;
  long long x_bs, y_bs;
  int x_pitch, y_pitch;
  int B, H, W, C, N, k, stride, pad_h, pad_w, dil_h, dil_w, Ho, Wo, M, Kt, act;
};

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == EVK_C2_RELU) return fmaxf(v, 0.f);
  if (act == EVK_C2_LRELU) return v >= 0.f ? v : 0.01f * v;
  if (act == EVK_C2_SIGMOID) return 1.f / (1.f + __expf(-v));
  if (act == EVK_C2_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

constexpr int STAGES = 3;
constexpr int SLAB = (BM + BN) * LDS;                        // floats of one pipeline stage: A [BM][LDS], B [BN][LDS]
constexpr int CONV_SMEM = STAGES * SLAB * 4;

// Stage K-slab k0 (columns k0 .. k0+31 of A = im2col(x) and of B = w) into smem with cp.async; out-of-image taps, rows past
// M, columns past Kt and output channels past N are zero-filled.  VEC: C, x_pitch, x_bs and Kt are multiples of 4 and the
// operands 16-byte aligned, so four consecutive k are four consecutive channels of one tap (one 16-byte copy); otherwise
// one 4-byte copy per element.
template <bool VEC>
__device__ __forceinline__ void load_slab(const ConvArgs& a, float* sA, float* sB, int k0, int m0, int n0,
                                          const long long* rbase, const int* riy, const int* rix) {
  const int tid = threadIdx.x;
  if (VEC) {
    const int kc = (tid & 7) * 4, rr = tid >> 3;            // 8 threads x 16 B cover a 32-column row
    const int k = k0 + kc;
    const bool kin = k < a.Kt;
    int c = 0, dy = 0, dx = 0;
    if (kin) {
      const int tap = k / a.C;
      c = k - tap * a.C;
      const int ky = tap / a.k;
      dy = ky * a.dil_h;
      dx = (tap - ky * a.k) * a.dil_w;
    }
#pragma unroll
    for (int i = 0; i < BM / 32; ++i) {
      const int r = rr + 32 * i;
      const int iy = riy[r] + dy, ix = rix[r] + dx;
      const bool ok = kin && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
      const float* src = ok ? a.x + rbase[r] + (long long)(iy * a.W + ix) * a.x_pitch + c : a.x;
      cp_async16(sA + r * LDS + kc, src, ok ? 16 : 0);
    }
#pragma unroll
    for (int j = 0; j < BN / 32; ++j) {
      const int n = n0 + rr + 32 * j;
      const bool ok = kin && n < a.N;
      cp_async16(sB + (rr + 32 * j) * LDS + kc, ok ? a.w + (long long)n * a.Kt + k : a.w, ok ? 16 : 0);
    }
  } else {
    const int kc = tid & 31, rr = tid >> 5;                 // one column per lane, one row per warp
    const int k = k0 + kc;
    const bool kin = k < a.Kt;
    int c = 0, dy = 0, dx = 0;
    if (kin) {
      const int tap = k / a.C;
      c = k - tap * a.C;
      const int ky = tap / a.k;
      dy = ky * a.dil_h;
      dx = (tap - ky * a.k) * a.dil_w;
    }
#pragma unroll 4
    for (int i = 0; i < BM / 8; ++i) {
      const int r = rr + 8 * i;
      const int iy = riy[r] + dy, ix = rix[r] + dx;
      const bool ok = kin && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
      const float* src = ok ? a.x + rbase[r] + (long long)(iy * a.W + ix) * a.x_pitch + c : a.x;
      cp_async4(sA + r * LDS + kc, src, ok ? 4 : 0);
    }
#pragma unroll 4
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + rr + 8 * j;
      const bool ok = kin && n < a.N;
      cp_async4(sB + (rr + 8 * j) * LDS + kc, ok ? a.w + (long long)n * a.Kt + k : a.w, ok ? 4 : 0);
    }
  }
}

template <bool PR, bool VEC>
__global__ void __launch_bounds__(NT, 2) conv2d_fwd_kernel(ConvArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ long long rbase[BM];
  __shared__ int riy[BM], rix[BM];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int HWo = a.Ho * a.Wo;
  if (tid < BM) {
    const int m = m0 + tid;
    if (m < a.M) {
      const int b = m / HWo, r = m - b * HWo, oy = r / a.Wo, ox = r - oy * a.Wo;
      rbase[tid] = (long long)b * a.x_bs;
      riy[tid] = oy * a.stride - a.pad_h;
      rix[tid] = ox * a.stride - a.pad_w;
    } else {
      rbase[tid] = 0; riy[tid] = -(1 << 29); rix[tid] = 0;      // never in bounds -> zero rows
    }
  }
  __syncthreads();

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;

  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int nk = (a.Kt + BKC - 1) / BKC;
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nk) load_slab<VEC>(a, smem + s * SLAB, smem + s * SLAB + BM * LDS, s * BKC, m0, n0, rbase, riy, rix);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();                 // slab kt landed for every thread; every thread is done with slab kt - 1
    {
      const int nx = kt + STAGES - 1, st = nx % STAGES;
      if (nx < nk) load_slab<VEC>(a, smem + st * SLAB, smem + st * SLAB + BM * LDS, nx * BKC, m0, n0, rbase, riy, rix);
      cp_async_commit();
    }
    const float* As = smem + (kt % STAGES) * SLAB;
    const float* Bs = As + BM * LDS;
    // 3xTF32: the tensor core's fp32 accumulation truncates, so each slab is summed from zero and added to acc in fp32
    float part[2][4][4];
    float (&sum)[2][4][4] = PR ? part : acc;
    if (PR) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.f;
    }
#pragma unroll
    for (int ks = 0; ks < BKC; ks += 8) {
      uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const float* p = As + (wm + mi * 16 + gq) * LDS + ks + t;
        const float v[4] = {p[0], p[8 * LDS], p[4], p[8 * LDS + 4]};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          ah[mi][q] = f2tf32(v[q]);
          if (PR) al[mi][q] = f2tf32(v[q] - __uint_as_float(ah[mi][q]));
        }
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float* p = Bs + (wn + ni * 8 + gq) * LDS + ks + t;
        const float v[2] = {p[0], p[4]};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          bh[ni][q] = f2tf32(v[q]);
          if (PR) bl[ni][q] = f2tf32(v[q] - __uint_as_float(bh[ni][q]));
        }
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          if (PR) {
            mma_tf32(sum[mi][ni], al[mi], bh[ni]);
            mma_tf32(sum[mi][ni], ah[mi], bl[ni]);
          }
          mma_tf32(sum[mi][ni], ah[mi], bh[ni]);
        }
    }
    if (PR) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[i][j][q] += part[i][j][q];
    }
  }
  cp_async_wait<0>();

  // epilogue: rows wm + mi*16 + gq (+8), columns wn + ni*8 + 2t (+1)
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm + mi * 16 + gq + 8 * h;
      if (m >= a.M) continue;
      const int b = m / HWo, r = m - b * HWo;
      float* yr = a.y + (long long)b * a.y_bs + (long long)r * a.y_pitch;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n0 + wn + ni * 8 + 2 * t + e;
          if (n >= a.N) continue;
          float v = acc[mi][ni][2 * h + e];
          if (a.scale) v *= __ldg(a.scale + n);
          if (a.bias) v += __ldg(a.bias + n);
          yr[n] = apply_act(v, a.act);
        }
    }
}

// ---- wgmma path (TF32, 16-byte-aligned operands): two consumer warpgroups, each 64 rows x BNW columns ----------------
// A and B slabs are K-major rows of 32 floats (128 B) in the 128-byte-swizzle layout of wgmma.cuh: chunk c of row r is
// stored at r * 128 + ((c ^ (r & 7)) << 4).  Every thread stages with cp.async (zero-fill as in load_slab), rounds what it
// staged to TF32 once it has landed, then makes the writes visible to the tensor core's async proxy before the barrier.
constexpr int WG_STAGES = 4;
template <int BNW>
constexpr int wg_stage_bytes() { return (BM + BNW) * BKC * 4; }
template <int BNW>
constexpr int wg_smem() { return WG_STAGES * wg_stage_bytes<BNW>() + 1024; }

template <int BNW>
__device__ __forceinline__ void load_slab_sw(const ConvArgs& a, uint32_t sA, uint32_t sB, int k0, int n0, const long long* rbase,
                                             const int* riy, const int* rix) {
  const int tid = threadIdx.x, ch = tid & 7, rr = tid >> 3;
  const int k = k0 + ch * 4;
  const bool kin = k < a.Kt;
  int c = 0, dy = 0, dx = 0;
  if (kin) {
    const int tap = k / a.C;
    c = k - tap * a.C;
    const int ky = tap / a.k;
    dy = ky * a.dil_h;
    dx = (tap - ky * a.k) * a.dil_w;
  }
#pragma unroll
  for (int i = 0; i < BM / 32; ++i) {
    const int r = rr + 32 * i;
    const int iy = riy[r] + dy, ix = rix[r] + dx;
    const bool ok = kin && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
    const float* src = ok ? a.x + rbase[r] + (long long)(iy * a.W + ix) * a.x_pitch + c : a.x;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sA + r * 128 + ((ch ^ (r & 7)) << 4)), "l"(src),
                 "r"(ok ? 16 : 0));
  }
#pragma unroll
  for (int j = 0; j < BNW / 32; ++j) {
    const int r = rr + 32 * j, n = n0 + r;
    const bool ok = kin && n < a.N;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sB + r * 128 + ((ch ^ (r & 7)) << 4)),
                 "l"(ok ? a.w + (long long)n * a.Kt + k : a.w), "r"(ok ? 16 : 0));
  }
}

// Round this thread's own chunks of a landed slab to TF32 in place (cvt.rna, as the mma.sync path rounds its fragments):
// the tensor core would otherwise truncate the fp32 operands, a bias that grows through the cascaded nets.
template <int BNW>
__device__ __forceinline__ void round_slab_tf32(uint32_t sA, uint32_t sB) {
  const int tid = threadIdx.x, ch = tid & 7, rr = tid >> 3;
#pragma unroll
  for (int i = 0; i < BM / 32 + BNW / 32; ++i) {
    const int r = rr + 32 * (i < BM / 32 ? i : i - BM / 32);
    const uint32_t addr = (i < BM / 32 ? sA : sB) + r * 128 + ((ch ^ (r & 7)) << 4);
    float v0, v1, v2, v3;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n" : "=f"(v0), "=f"(v1), "=f"(v2), "=f"(v3) : "r"(addr));
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(f2tf32(v0)), "r"(f2tf32(v1)), "r"(f2tf32(v2)),
                 "r"(f2tf32(v3)) : "memory");
  }
}

template <int BNW>
__global__ void __launch_bounds__(NT, 1) conv2d_fwd_wgmma_kernel(ConvArgs a) {
  extern __shared__ __align__(16) unsigned char wsm[];
  __shared__ long long rbase[BM];
  __shared__ int riy[BM], rix[BM];
  const int tid = threadIdx.x, wg = tid >> 7, tw = tid & 127;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BNW;
  const int HWo = a.Ho * a.Wo;
  if (tid < BM) {
    const int m = m0 + tid;
    if (m < a.M) {
      const int b = m / HWo, r = m - b * HWo, oy = r / a.Wo, ox = r - oy * a.Wo;
      rbase[tid] = (long long)b * a.x_bs;
      riy[tid] = oy * a.stride - a.pad_h;
      rix[tid] = ox * a.stride - a.pad_w;
    } else {
      rbase[tid] = 0; riy[tid] = -(1 << 29); rix[tid] = 0;
    }
  }
  __syncthreads();
  const uint32_t base = (smem_u32(wsm) + 1023u) & ~1023u;   // swizzle atoms are 1024-byte aligned
  constexpr uint32_t SB = wg_stage_bytes<BNW>();
  float acc[BNW / 2];
#pragma unroll
  for (int i = 0; i < BNW / 2; ++i) acc[i] = 0.f;

  const int nk = (a.Kt + BKC - 1) / BKC;
#pragma unroll
  for (int s = 0; s < WG_STAGES - 1; ++s) {
    if (s < nk) load_slab_sw<BNW>(a, base + s * SB, base + s * SB + BM * 128, s * BKC, n0, rbase, riy, rix);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<WG_STAGES - 2>();
    {
      const uint32_t sa = base + (kt % WG_STAGES) * SB;
      round_slab_tf32<BNW>(sa, sa + BM * 128);
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();                  // slab kt visible to the tensor core; slab kt - 1 no longer read (waited below)
    {
      const int nx = kt + WG_STAGES - 1;
      const uint32_t st = base + (nx % WG_STAGES) * SB;
      if (nx < nk) load_slab_sw<BNW>(a, st, st + BM * 128, nx * BKC, n0, rbase, riy, rix);
      cp_async_commit();
    }
    const uint32_t sa = base + (kt % WG_STAGES) * SB;
    const uint64_t da = wg_desc_sw128(sa + wg * 64 * 128), db = wg_desc_sw128(sa + BM * 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BKC / 8; ++ks) wgmma_tf32<BNW>(acc, da + 2 * ks, db + 2 * ks, 1u);   // +32 B per K step
    wgmma_commit();
    wgmma_wait<0>();
  }
  cp_async_wait<0>();

  // thread tw holds rows 16 (tw / 32) + (tw % 32) / 4 (+ 8) and columns 8 j + 2 (tw % 4) (+ 1): acc[4 j + 2 h + e]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + wg * 64 + 16 * (tw >> 5) + ((tw & 31) >> 2) + 8 * h;
    if (m >= a.M) continue;
    const int b = m / HWo, r = m - b * HWo;
    float* yr = a.y + (long long)b * a.y_bs + (long long)r * a.y_pitch;
#pragma unroll
    for (int j = 0; j < BNW / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (tw & 3) + e;
        if (n >= a.N) continue;
        float v = acc[4 * j + 2 * h + e];
        if (a.scale) v *= __ldg(a.scale + n);
        if (a.bias) v += __ldg(a.bias + n);
        yr[n] = apply_act(v, a.act);
      }
  }
}

template <int BNW>
int launch_conv_wgmma(const ConvArgs& a, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv2d_fwd_wgmma_kernel<BNW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         wg_smem<BNW>());
    EVK_REQUIRE(e == cudaSuccess, EVK_ERR_CUDA, "conv2d: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  dim3 grid(cdiv(a.M, BM), cdiv(a.N, BNW));
  EVK_REQUIRE(grid.y <= 65535, EVK_ERR_ARG, "conv2d: too many output channels");
  conv2d_fwd_wgmma_kernel<BNW><<<grid, NT, wg_smem<BNW>(), st>>>(a);
  return check_launch("conv2d_fwd_wgmma");
}

template <bool PR, bool VEC>
int launch_conv(const ConvArgs& a, dim3 grid, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv2d_fwd_kernel<PR, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, CONV_SMEM);
    EVK_REQUIRE(e == cudaSuccess, EVK_ERR_CUDA, "conv2d: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  conv2d_fwd_kernel<PR, VEC><<<grid, NT, CONV_SMEM, st>>>(a);
  return check_launch("conv2d_fwd");
}

// one thread per output element, channel fastest
__global__ void dwconv3x3_kernel(const float* __restrict__ x, int x_pitch, long long x_bs, const float* __restrict__ w,
                                 float* __restrict__ y, int y_pitch, long long y_bs, int B, int H, int W, int C, int dil) {
  const long long total = (long long)B * H * W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long p = i / C;
    const int ox = (int)(p % W); p /= W;
    const int oy = (int)(p % H);
    const int b = (int)(p / H);
    const float* xb = x + (long long)b * x_bs + c;
    float s = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy + (ky - 1) * dil;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox + (kx - 1) * dil;
        if (ix < 0 || ix >= W) continue;
        s = fmaf(__ldg(w + c * 9 + ky * 3 + kx), __ldg(xb + (long long)(iy * W + ix) * x_pitch), s);
      }
    }
    y[(long long)b * y_bs + (long long)(oy * W + ox) * y_pitch + c] = s;
  }
}

// PyTorch's align_corners=True source index: scale = (in - 1) / (out - 1) in fp32, src = scale * dst, i1 = i0 + (i0 < in - 1)
__device__ __forceinline__ void ac_index(int o, int in, int out, int& i0, int& i1, float& l1) {
  const float sc = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  const float src = sc * (float)o;
  i0 = min((int)src, in - 1);
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = src - (float)i0;
}

__global__ void resize_ac_kernel(const float* __restrict__ x, int x_pitch, long long x_bs, int Hi, int Wi,
                                 float* __restrict__ y, int y_pitch, long long y_bs, int Ho, int Wo, int B, int C) {
  const long long total = (long long)B * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long p = i / C;
    const int ox = (int)(p % Wo); p /= Wo;
    const int oy = (int)(p % Ho);
    const int b = (int)(p / Ho);
    int h0, h1, w0, w1;
    float lh, lw;
    ac_index(oy, Hi, Ho, h0, h1, lh);
    ac_index(ox, Wi, Wo, w0, w1, lw);
    const float* xb = x + (long long)b * x_bs + c;
    const float v00 = __ldg(xb + (long long)(h0 * Wi + w0) * x_pitch), v01 = __ldg(xb + (long long)(h0 * Wi + w1) * x_pitch);
    const float v10 = __ldg(xb + (long long)(h1 * Wi + w0) * x_pitch), v11 = __ldg(xb + (long long)(h1 * Wi + w1) * x_pitch);
    const float hl0 = 1.f - lh, wl0 = 1.f - lw;
    y[(long long)b * y_bs + (long long)(oy * Wo + ox) * y_pitch + c] = hl0 * (wl0 * v00 + lw * v01) + lh * (wl0 * v10 + lw * v11);
  }
}

// y[b][0][x][c] = mean over rows of x[b][:][x][c]; rows are added in order
__global__ void mean_h_kernel(const float* __restrict__ x, int x_pitch, long long x_bs, float* __restrict__ y, int B, int H,
                              int W, int C) {
  const long long total = (long long)B * W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long p = i / C;
    const int ox = (int)(p % W), b = (int)(p / W);
    const float* xb = x + (long long)b * x_bs + (long long)ox * x_pitch + c;
    float s = 0.f;
    for (int r = 0; r < H; ++r) s += __ldg(xb + (long long)r * W * x_pitch);
    y[i] = s / (float)H;
  }
}

__global__ void vr_mask_head_kernel(const float* __restrict__ h, int h_pitch, long long h_bs, const float* __restrict__ w,
                                    int Ch, const float* __restrict__ mix, float* __restrict__ out, int B, int max_bin,
                                    int out_bin, int W, int offset, int split_bin, float e_lo, float e_hi, int use_agg) {
  const int Wc = W - 2 * offset;
  const long long total = (long long)B * out_bin * Wc;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xo = (int)(i % Wc);
    const long long p = i / Wc;
    const int row = (int)(p % out_bin), b = (int)(p / out_bin);
    const int x = xo + offset, hr = min(row, max_bin - 1);          // replicate pad past max_bin
    const float* hp = h + (long long)b * h_bs + (long long)(hr * W + x) * h_pitch;
    float s0 = 0.f, s1 = 0.f;
    for (int k = 0; k < Ch; ++k) {
      const float v = __ldg(hp + k);
      s0 = fmaf(__ldg(w + k), v, s0);
      s1 = fmaf(__ldg(w + Ch + k), v, s1);
    }
    float m0 = 1.f / (1.f + expf(-s0)), m1 = 1.f / (1.f + expf(-s1));
    if (use_agg) {
      const float e = row < split_bin ? e_lo : e_hi;
      m0 = powf(m0, e); m1 = powf(m1, e);
    }
    const long long plane = (long long)out_bin * W, oplane = (long long)out_bin * Wc;
    const float* mx = mix + (long long)b * 2 * plane + (long long)row * W + x;
    float* o = out + (long long)b * 2 * oplane + (long long)row * Wc + xo;
    o[0] = m0 * __ldg(mx);
    o[oplane] = m1 * __ldg(mx + plane);
  }
}

inline int grid_for(long long total) {
  const long long g = (total + 255) / 256;
  return (int)(g < 32LL * kNumSMs ? g : 32LL * kNumSMs);
}

}  // namespace
extern int g_precise;
}  // namespace evk

using namespace evk;

extern "C" int evk_conv2d_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, const float* scale,
                              const float* bias, float* y, int32_t y_pitch, int64_t y_bs, int32_t B, int32_t H, int32_t W,
                              int32_t C, int32_t N, int32_t k, int32_t stride, int32_t pad_h, int32_t pad_w, int32_t dil_h,
                              int32_t dil_w, int32_t act, cudaStream_t st) {
  EVK_REQUIRE(x && w && y, EVK_ERR_ARG, "conv2d: null tensor");
  EVK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && N > 0, EVK_ERR_ARG, "conv2d: bad sizes B=%d H=%d W=%d C=%d N=%d", B, H, W,
              C, N);
  EVK_REQUIRE((k >= 1 && k <= 3) && (stride == 1 || stride == 2) && pad_h >= 0 && pad_w >= 0 && dil_h >= 1 && dil_w >= 1,
              EVK_ERR_ARG, "conv2d: kernel %d stride %d pad (%d, %d) dilation (%d, %d) (kernel 1, 2 or 3, stride 1 or 2)", k,
              stride, pad_h, pad_w, dil_h, dil_w);
  EVK_REQUIRE(act >= EVK_C2_NONE && act <= EVK_C2_GELU, EVK_ERR_ARG, "conv2d: bad activation %d", act);
  EVK_REQUIRE(x_pitch >= C && y_pitch >= N, EVK_ERR_ARG, "conv2d: pitch smaller than the channel count");
  const int span_h = dil_h * (k - 1) + 1, span_w = dil_w * (k - 1) + 1;
  EVK_REQUIRE(H + 2 * pad_h >= span_h && W + 2 * pad_w >= span_w, EVK_ERR_ARG, "conv2d: input smaller than the kernel");
  const int Ho = (H + 2 * pad_h - span_h) / stride + 1, Wo = (W + 2 * pad_w - span_w) / stride + 1;
  const long long M = (long long)B * Ho * Wo, Kt = (long long)k * k * C;
  EVK_REQUIRE(M < (1ll << 31) && Kt < (1ll << 31) && (long long)N * Kt < (1ll << 31) && (long long)H * W < (1 << 30),
              EVK_ERR_ARG, "conv2d: problem too large");
  ConvArgs a{x, w, scale, bias, y, x_bs, y_bs, x_pitch, y_pitch, B, H, W, C, N, k, stride,
             pad_h, pad_w, dil_h, dil_w, Ho, Wo, (int)M, (int)Kt, act};
  dim3 grid(cdiv(M, BM), cdiv(N, BN));
  EVK_REQUIRE(grid.y <= 65535, EVK_ERR_ARG, "conv2d: too many output channels");
  const bool vec = C % 4 == 0 && x_pitch % 4 == 0 && x_bs % 4 == 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)w % 16 == 0;
  // 3xTF32 splits the operands in registers, so it runs on mma.sync; so do operands the 16-byte copies cannot read
  if (g_precise) return vec ? launch_conv<true, true>(a, grid, st) : launch_conv<true, false>(a, grid, st);
  if (!vec) return launch_conv<false, false>(a, grid, st);
  if (N <= 32) return launch_conv_wgmma<32>(a, st);
  if (N <= 64) return launch_conv_wgmma<64>(a, st);
  return launch_conv_wgmma<128>(a, st);
}

extern "C" int evk_dwconv3x3_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, float* y, int32_t y_pitch,
                                 int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t dil, cudaStream_t st) {
  EVK_REQUIRE(x && w && y, EVK_ERR_ARG, "dwconv3x3: null tensor");
  EVK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && dil >= 1 && x_pitch >= C && y_pitch >= C, EVK_ERR_ARG,
              "dwconv3x3: bad sizes B=%d H=%d W=%d C=%d dil=%d", B, H, W, C, dil);
  const long long total = (long long)B * H * W * C;
  dwconv3x3_kernel<<<grid_for(total), 256, 0, st>>>(x, x_pitch, x_bs, w, y, y_pitch, y_bs, B, H, W, C, dil);
  return check_launch("dwconv3x3");
}

extern "C" int evk_resize_bilinear_ac(const float* x, int32_t x_pitch, int64_t x_bs, int32_t Hi, int32_t Wi, float* y,
                                      int32_t y_pitch, int64_t y_bs, int32_t Ho, int32_t Wo, int32_t B, int32_t C,
                                      cudaStream_t st) {
  EVK_REQUIRE(x && y, EVK_ERR_ARG, "resize: null tensor");
  EVK_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0 && x_pitch >= C && y_pitch >= C, EVK_ERR_ARG,
              "resize: bad sizes B=%d %dx%d -> %dx%d C=%d", B, Hi, Wi, Ho, Wo, C);
  const long long total = (long long)B * Ho * Wo * C;
  resize_ac_kernel<<<grid_for(total), 256, 0, st>>>(x, x_pitch, x_bs, Hi, Wi, y, y_pitch, y_bs, Ho, Wo, B, C);
  return check_launch("resize_bilinear_ac");
}

extern "C" int evk_mean_h(const float* x, int32_t x_pitch, int64_t x_bs, float* y, int32_t B, int32_t H, int32_t W, int32_t C,
                          cudaStream_t st) {
  EVK_REQUIRE(x && y, EVK_ERR_ARG, "mean_h: null tensor");
  EVK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && x_pitch >= C, EVK_ERR_ARG, "mean_h: bad sizes");
  const long long total = (long long)B * W * C;
  mean_h_kernel<<<grid_for(total), 256, 0, st>>>(x, x_pitch, x_bs, y, B, H, W, C);
  return check_launch("mean_h");
}

extern "C" int evk_vr_mask_head(const float* h, int32_t h_pitch, int64_t h_bs, const float* w, int32_t Ch, const float* mix,
                                float* out, int32_t B, int32_t max_bin, int32_t out_bin, int32_t W, int32_t offset,
                                int32_t split_bin, float e_lo, float e_hi, int32_t use_agg, cudaStream_t st) {
  EVK_REQUIRE(h && w && mix && out, EVK_ERR_ARG, "vr_mask_head: null tensor");
  EVK_REQUIRE(B > 0 && Ch > 0 && h_pitch >= Ch && max_bin > 0 && out_bin >= max_bin && offset >= 0 && W > 2 * offset,
              EVK_ERR_ARG, "vr_mask_head: bad sizes B=%d Ch=%d max_bin=%d out_bin=%d W=%d offset=%d", B, Ch, max_bin,
              out_bin, W, offset);
  const long long total = (long long)B * out_bin * (W - 2 * offset);
  vr_mask_head_kernel<<<grid_for(total), 256, 0, st>>>(h, h_pitch, h_bs, w, Ch, mix, out, B, max_bin, out_bin, W, offset,
                                                       split_bin, e_lo, e_hi, use_agg);
  return check_launch("vr_mask_head");
}
