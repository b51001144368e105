// Direct (CUDA-core) generalised convolution for skinny layers: 1-channel inputs, 1-channel outputs and
// the grouped k=41 convs of DiscriminatorS (4 in-channels per group).  These layers are bandwidth /
// latency bound (K = Q*C/G <= 164 or N == 1); tensor-core tiles would be >90% padding.
// Same operator and descriptor as gconv.cu; W is [Q][N][C/G] (pitch ldw).
#include "evk_common.cuh"

namespace evk {

struct DP {
  const float* x; float* w; float* y; const float* res; const float* bias;
  const int* in_len; const int* out_len;
  long long x_sb, x_sh, w_sb, w_sh, w_sq, y_sb, y_sh, r_sb, r_sh;
  int ldx, ldw, ldy, ldr;
  int Z, H, C, N, Q, G, Tin, J, P, is, os, o0, Tout, act;
  float slope;
  int chunk;
  int off[EVK_MAX_TAPS];
};

__device__ __forceinline__ float dact(float v, int act, float slope) {
  if (act == EVK_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == EVK_ACT_RELU) return fmaxf(v, 0.f);
  if (act == EVK_ACT_TANH) return tanhf(v);
  if (act == EVK_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

// one thread per output element (pos, n), n fastest
__global__ void direct_fwd_thread(const __grid_constant__ DP p) {
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const long long npos = (long long)p.J * p.P;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= npos * p.N) return;
  const int n = (int)(idx % p.N);
  const long long pos = idx / p.N;
  const int j = (int)(pos / p.P), w = (int)(pos - (long long)j * p.P);
  const int Cg = p.C / p.G, Ng = p.N / p.G, g = n / Ng;
  const float* X = p.x + b * p.x_sb + h * p.x_sh + g * Cg;
  const float* W = p.w + b * p.w_sb + h * p.w_sh + (long long)n * p.ldw;
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  float acc = 0.f;
  for (int q = 0; q < p.Q; ++q) {
    const int ij = j * p.is + p.off[q];
    if (ij < 0 || ij >= lim) continue;
    const float* xr = X + ((long long)ij * p.P + w) * p.ldx;
    const float* wr = W + (long long)q * p.w_sq;
    for (int c = 0; c < Cg; ++c) acc = fmaf(xr[c], wr[c], acc);
  }
  const int oj = p.o0 + j * p.os;
  const long long orow = (long long)oj * p.P + w;
  if (p.bias) acc += p.bias[n];
  if (p.res) acc += (p.res + b * p.r_sb + h * p.r_sh)[orow * p.ldr + n];
  acc = dact(acc, p.act, p.slope);
  if (p.out_len && oj >= p.out_len[b]) acc = 0.f;
  (p.y + b * p.y_sb + h * p.y_sh)[orow * p.ldy + n] = acc;
}

// one warp per output element (large K = Q*Cg, e.g. 1024->1 k3)
__global__ void direct_fwd_warp(const __grid_constant__ DP p) {
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const long long npos = (long long)p.J * p.P;
  const long long idx = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (idx >= npos * p.N) return;
  const int n = (int)(idx % p.N);
  const long long pos = idx / p.N;
  const int j = (int)(pos / p.P), w = (int)(pos - (long long)j * p.P);
  const int Cg = p.C / p.G, Ng = p.N / p.G, g = n / Ng;
  const float* X = p.x + b * p.x_sb + h * p.x_sh + g * Cg;
  const float* W = p.w + b * p.w_sb + h * p.w_sh + (long long)n * p.ldw;
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  float acc = 0.f;
  for (int q = 0; q < p.Q; ++q) {
    const int ij = j * p.is + p.off[q];
    if (ij < 0 || ij >= lim) continue;
    const float* xr = X + ((long long)ij * p.P + w) * p.ldx;
    const float* wr = W + (long long)q * p.w_sq;
    for (int c = lane; c < Cg; c += 32) acc = fmaf(xr[c], wr[c], acc);
  }
  acc = warp_sum(acc);
  if (lane) return;
  const int oj = p.o0 + j * p.os;
  const long long orow = (long long)oj * p.P + w;
  if (p.bias) acc += p.bias[n];
  if (p.res) acc += (p.res + b * p.r_sb + h * p.r_sh)[orow * p.ldr + n];
  acc = dact(acc, p.act, p.slope);
  if (p.out_len && oj >= p.out_len[b]) acc = 0.f;
  (p.y + b * p.y_sb + h * p.y_sh)[orow * p.ldy + n] = acc;
}

// dX[ipos][c] = sum_q sum_{n in group} dY[orow(j)][n] * W[q][n][c_local],  j*is + off[q] == ij
__global__ void direct_dgrad(const __grid_constant__ DP p) {
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const long long nin = (long long)p.Tin * p.P;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nin * p.C) return;
  const int c = (int)(idx % p.C);
  const long long ipos = idx / p.C;
  const int ij = (int)(ipos / p.P), w = (int)(ipos - (long long)ij * p.P);
  const int Cg = p.C / p.G, Ng = p.N / p.G, g = c / Cg, cl = c - g * Cg;
  const float* Yg = p.y + b * p.y_sb + h * p.y_sh + g * Ng;
  const float* W = p.w + b * p.w_sb + h * p.w_sh + (long long)(g * Ng) * p.ldw + cl;
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  float acc = 0.f;
  if (ij < lim) {
    for (int q = 0; q < p.Q; ++q) {
      const int t = ij - p.off[q];
      if (t < 0) continue;
      const int j = t / p.is;
      if (j * p.is != t || j >= p.J) continue;
      const float* yr = Yg + ((long long)(p.o0 + j * p.os) * p.P + w) * p.ldy;
      const float* wr = W + (long long)q * p.w_sq;
      for (int n = 0; n < Ng; ++n) acc = fmaf(yr[n], wr[(long long)n * p.ldw], acc);
    }
  }
  (const_cast<float*>(p.x) + b * p.x_sb + h * p.x_sh)[ipos * p.ldx + c] = acc;
}

// dW[q][n][cl] += sum_z sum_pos dY[orow][n] * X[irow][g*Cg+cl]; one thread per weight, positions chunked over grid.x.
// Each (z, chunk) writes its partial to part[(z * chunks + chunk) * nw + widx]; ordered_sum adds them in that order.
__global__ void direct_wgrad(const __grid_constant__ DP p, float* __restrict__ part) {
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const int Cg = p.C / p.G, Ng = p.N / p.G;
  const long long nw = (long long)p.Q * p.N * Cg;
  const long long widx = (long long)blockIdx.y * blockDim.x + threadIdx.x;
  if (widx >= nw) return;
  const int cl = (int)(widx % Cg);
  const int n = (int)((widx / Cg) % p.N);
  const int q = (int)(widx / ((long long)Cg * p.N));
  const int g = n / Ng;
  const float* X = p.x + b * p.x_sb + h * p.x_sh + g * Cg + cl;
  const float* Yg = p.y + b * p.y_sb + h * p.y_sh + n;
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  const long long npos = (long long)p.J * p.P;
  const long long pbeg = (long long)blockIdx.x * p.chunk, pend = min(npos, pbeg + p.chunk);
  const int offq = p.off[q];
  float acc = 0.f;
  for (long long pos = pbeg; pos < pend; ++pos) {
    const int j = (int)(pos / p.P), w = (int)(pos - (long long)j * p.P);
    const int ij = j * p.is + offq;
    if (ij < 0 || ij >= lim) continue;
    acc = fmaf(Yg[((long long)(p.o0 + j * p.os) * p.P + w) * p.ldy], X[((long long)ij * p.P + w) * p.ldx], acc);
  }
  part[((long long)z * gridDim.x + blockIdx.x) * nw + widx] = acc;
}

static int fill_dp(const evk_gconv_desc* d, DP& p) {
  EVK_REQUIRE(d != nullptr, EVK_ERR_ARG, "conv_direct: null descriptor");
  EVK_REQUIRE(d->Q >= 1 && d->Q <= EVK_MAX_TAPS, EVK_ERR_ARG, "conv_direct: Q=%d out of range", d->Q);
  const int G = d->G < 1 ? 1 : d->G;
  EVK_REQUIRE(d->C % G == 0 && d->N % G == 0, EVK_ERR_ARG, "conv_direct: C=%d N=%d not divisible by G=%d", d->C, d->N, G);
  EVK_REQUIRE(d->Z >= 1 && d->H >= 1 && d->P >= 1 && d->is >= 1 && d->os >= 1, EVK_ERR_ARG, "conv_direct: bad sizes");
  p.x = d->x; p.w = d->w; p.y = d->y; p.res = d->res; p.bias = d->bias; p.in_len = d->in_len; p.out_len = d->out_len;
  p.x_sb = d->x_sb; p.x_sh = d->x_sh; p.w_sb = d->w_sb; p.w_sh = d->w_sh; p.w_sq = d->w_sq;
  p.y_sb = d->y_sb; p.y_sh = d->y_sh; p.r_sb = d->r_sb; p.r_sh = d->r_sh;
  p.ldx = d->ldx; p.ldw = d->ldw; p.ldy = d->ldy; p.ldr = d->ldr;
  p.Z = d->Z; p.H = d->H; p.C = d->C; p.N = d->N; p.Q = d->Q; p.G = G; p.Tin = d->Tin; p.J = d->J; p.P = d->P;
  p.is = d->is; p.os = d->os; p.o0 = d->o0; p.Tout = d->Tout; p.act = d->act; p.slope = d->slope; p.chunk = 0;
  for (int i = 0; i < EVK_MAX_TAPS; ++i) p.off[i] = i < d->Q ? d->off[i] : 0;
  if (d->J > 0) {
    long long last = (long long)d->o0 + (long long)(d->J - 1) * d->os;
    EVK_REQUIRE(d->o0 >= 0 && last < d->Tout, EVK_ERR_ARG, "conv_direct: output positions exceed Tout");
  }
  return EVK_OK;
}

}  // namespace evk
using namespace evk;

extern "C" int evk_conv_direct_fwd(const evk_gconv_desc* d, evk_stream_t stream) {
  DP p;
  int rc = fill_dp(d, p);
  if (rc) return rc;
  const long long total = (long long)p.J * p.P * p.N;
  if (total == 0) return EVK_OK;
  const int K = p.Q * (p.C / p.G);
  if (K >= 512) {
    dim3 grid(cdiv(total * 32, 256), 1, p.Z);
    direct_fwd_warp<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  } else {
    dim3 grid(cdiv(total, 256), 1, p.Z);
    direct_fwd_thread<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  }
  g_disp_flops[3] += desc_flops(d);
  return check_launch("conv_direct_fwd");
}

extern "C" int evk_conv_direct_dgrad(const evk_gconv_desc* d, evk_stream_t stream) {
  DP p;
  int rc = fill_dp(d, p);
  if (rc) return rc;
  const long long total = (long long)p.Tin * p.P * p.C;
  if (total == 0) return EVK_OK;
  dim3 grid(cdiv(total, 256), 1, p.Z);
  direct_dgrad<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  g_disp_flops[3] += desc_flops(d);
  return check_launch("conv_direct_dgrad");
}

extern "C" int evk_conv_direct_wgrad(const evk_gconv_desc* d, evk_stream_t stream) {
  DP p;
  int rc = fill_dp(d, p);
  if (rc) return rc;
  const long long nw = (long long)p.Q * p.N * (p.C / p.G);
  const long long npos = (long long)p.J * p.P;
  if (nw == 0 || npos == 0) return EVK_OK;
  const int wblocks = cdiv(nw, 256);
  long long want = ((long long)kNumSMs * 8 + (long long)wblocks * p.Z - 1) / ((long long)wblocks * p.Z);
  long long chunk = (npos + want - 1) / want;
  if (chunk < 128) chunk = 128;
  p.chunk = (int)chunk;
  dim3 grid(cdiv(npos, chunk), wblocks, p.Z);
  EVK_REQUIRE(grid.y <= 65535, EVK_ERR_ARG, "conv_direct_wgrad: too many weights");
  const int chunks = (int)grid.x, Cg = p.C / p.G;
  Scratch part_buf(nw * chunks * p.Z, (cudaStream_t)stream);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "conv_direct_wgrad: scratch allocation failed");
  direct_wgrad<<<grid, 256, 0, (cudaStream_t)stream>>>(p, part);
  g_disp_flops[6] += desc_flops(d);
  if (int rc2 = check_launch("conv_direct_wgrad")) return rc2;
  if (p.w_sb == 0 && p.w_sh == 0)                                  // one weight for every z: all partials in (z, chunk) order
    return ordered_sum(part, p.Z * chunks, p.Q, p.N, Cg, p.w, p.w_sq, p.ldw, (cudaStream_t)stream);
  for (int z = 0; z < p.Z; ++z) {                                  // z in order, each adding its chunks
    const int b = z / p.H, h = z - b * p.H;
    if (int rc2 = ordered_sum(part + (long long)z * chunks * nw, chunks, p.Q, p.N, Cg, p.w + b * p.w_sb + h * p.w_sh, p.w_sq, p.ldw,
                              (cudaStream_t)stream))
      return rc2;
  }
  return EVK_OK;
}
