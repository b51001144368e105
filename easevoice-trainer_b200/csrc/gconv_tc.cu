// wgmma implicit-GEMM convolution (sm_90a): the stride-1 launches of the generalised conv
//
//   Y[z][pos][n] = epi( sum_q sum_c X[z][pos + off[q]*P][c] * W[z][q][n][c] ),   pos = j*P + w  (is == 1)
//
// Mapping: 128 output positions per M tile = two warpgroups x 64 rows (wgmma M), output channels = wgmma N, input
// channels = K.  Both operands are K-major in the canonical *interleaved* (no-swizzle) core-matrix layout: for every
// 16-byte K-chunk a panel [rows][16 B].  A row shift is then a plain +16 B*rows start-address offset, so ONE staged slab
// of input rows serves every tap (the smem descriptor of tap q just starts off[q]*P rows further down) -- the implicit
// im2col costs no extra shared-memory fill.  Accumulators live in registers (fp32, MT x BN / 2 per thread).
// Activations are staged global -> registers -> cvt.rna.tf32 -> smem (round-to-nearest instead of the tensor
// core's operand truncation, which would bias every product towards zero); weights are pre-rounded at pack time.
#include "wgmma.cuh"

namespace evk {

struct TP : ConvP {
  int TG, NG;               // taps per group, groups
  int slab_rows, a_pitch;   // rows staged per chunk, slab panel pitch (rows, == 4 mod 8)
  int KCH;                  // 16-byte K-chunks per stage (2, 4 or 8)
};

constexpr int TC_THREADS = 256;                       // two warpgroups

// BN: N tile (wgmma N); MT: number of 128-position M tiles per CTA (weights reused MT times)
template <int BN, int MT>
__global__ void __launch_bounds__(TC_THREADS, 1) gconv_tc_kernel(const __grid_constant__ TP p) {
  constexpr int B_PITCH = BN + 4;                               // weight panel pitch (rows); == 4 (mod 8)
  extern __shared__ __align__(128) uint8_t tsm[];
  const int KCH = p.KCH, KC = KCH * 4;
  const int slab_bytes = KCH * p.a_pitch * 16;
  const int wt_bytes = p.TG * KCH * B_PITCH * 16;
  uint8_t* slab0 = tsm;                                         // [2][KCH][a_pitch][16 B]
  uint8_t* wt0 = tsm + 2 * slab_bytes;                          // [NW][TG][KCH][B_PITCH][16 B]
  constexpr int NW = 2;                                         // weight-stage ring depth

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;                                     // warpgroup: rows 64 wg .. 64 wg + 63 of each M tile
  const int z = blockIdx.z, b = z / p.H, h = z - b * p.H;
  const float* X = p.x + b * p.x_sb + h * p.x_sh;
  const float* Wg = p.w + b * p.w_sb + h * p.w_sh;
  const int p0 = blockIdx.x * (MT * 128), n0 = blockIdx.y * BN;
  const int npos = p.J * p.P;
  const int lo = p0 + p.off_min * p.P;                          // flat input row of slab row 0
  int lim = p.Tin;
  if (p.in_len) lim = min(lim, p.in_len[b]);
  const int lim_rows = lim * p.P;

  const int nchunks = (p.C + KC - 1) / KC;
  const int U = nchunks * p.NG;

  auto load_slab = [&](int ch, int buf) {                       // global -> regs -> rna(tf32) -> smem panels
    uint8_t* dst = slab0 + buf * slab_bytes;
    const int c0 = ch * KC;
    const int total = p.slab_rows * KCH;
    for (int i = tid; i < total; i += TC_THREADS) {
      const int r = i / KCH, kc = i - r * KCH;
      const int c = c0 + kc * 4, f = lo + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f >= 0 && f < lim_rows && c < p.C) v = *reinterpret_cast<const float4*>(X + (long long)f * p.ldx + c);
      uint4 t = make_uint4(f2tf32(v.x), f2tf32(v.y), f2tf32(v.z), f2tf32(v.w));
      *reinterpret_cast<uint4*>(dst + ((size_t)kc * p.a_pitch + r) * 16) = t;
    }
  };
  auto load_w = [&](int ch, int g, int buf) {                   // cp.async (weights are tf32-rounded at pack time)
    uint8_t* dst = wt0 + buf * wt_bytes;
    const int c0 = ch * KC;
    const int total = p.TG * BN * KCH;
    for (int i = tid; i < total; i += TC_THREADS) {
      const int tq = i / (BN * KCH), rem = i - tq * (BN * KCH);
      const int n = rem / KCH, kc = rem - n * KCH;
      const int c = c0 + kc * 4, q = g * p.TG + tq;
      const bool ok = (q < p.Q) && (n0 + n < p.N) && (c < p.C);
      const float* src = ok ? (Wg + (long long)q * p.w_sq + (long long)(n0 + n) * p.ldw + c) : Wg;
      cp_async16(dst + ((size_t)(tq * KCH + kc) * B_PITCH + n) * 16, src, ok ? 16 : 0);
    }
  };

  float acc[MT][BN / 2];
  load_slab(0, 0);
  load_w(0, 0, 0);
  cp_async_commit();
  // Pipeline: unit u reads weight stage u % 2 and slab buffer ch % 2.  Its wgmmas are issued first; the loads of unit u+1
  // (the other weight stage and, at a chunk boundary, the other slab buffer) run while they execute.  Both buffers were
  // last read by unit u-1, whose wgmmas every thread waited for before the barrier that opens unit u.
  for (int u = 0; u < U; ++u) {
    const int ch = u / p.NG, g = u - ch * p.NG;
    cp_async_wait<0>();
    asm volatile("fence.proxy.async.shared::cta;\n");           // generic-proxy smem writes -> visible to the tensor core
    __syncthreads();
    {
      const uint32_t sl = smem_u32(slab0 + (ch & 1) * slab_bytes) + (uint32_t)(wg * 64 * 16);
      const uint32_t wt = smem_u32(wt0 + (u % NW) * wt_bytes);
      const int ntaps = min(p.TG, p.Q - g * p.TG);
      wgmma_fence();
      for (int tq = 0; tq < ntaps; ++tq) {
        const int toff = (p.off[g * p.TG + tq] - p.off_min) * p.P;
        for (int k2 = 0; k2 < KCH / 2; ++k2) {
          const uint64_t bdesc = wg_desc_plain(wt + ((tq * KCH + 2 * k2) * B_PITCH) * 16, B_PITCH * 16, 128);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) {
            const uint64_t adesc = wg_desc_plain(sl + ((2 * k2) * p.a_pitch + mt * 128 + toff) * 16, p.a_pitch * 16, 128);
            wgmma_tf32<BN>(acc[mt], adesc, bdesc, (u | tq | k2) != 0 ? 1u : 0u);
          }
        }
      }
      wgmma_commit();
    }
    if (u + 1 < U) {
      const int ch1 = (u + 1) / p.NG, g1 = (u + 1) - ch1 * p.NG;
      if (g1 == 0) load_slab(ch1, ch1 & 1);
      load_w(ch1, g1, (u + 1) % NW);
      cp_async_commit();
    }
    wgmma_wait<0>();
  }

  float* Y = p.y + b * p.y_sb + h * p.y_sh;
  const float* R = p.res ? (p.res + b * p.r_sb + h * p.r_sh) : nullptr;
  const float* bias = p.bias ? (p.bias + h * p.b_sh) : nullptr;
  const int olen = p.out_len ? p.out_len[b] : 0x7fffffff;
  // accumulator fragment: d[4j + 2hh + e] = (row 16 (warp % 4) + lane / 4 + 8 hh, column 8 j + 2 (lane % 4) + e)
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int pos = p0 + mt * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hh;
      if (pos >= npos) continue;
      const int j = pos / p.P, w = pos - j * p.P;
      const int oj = p.o0 + j * p.os;
      const long long orow = (long long)oj * p.P + w;
      const bool live = oj < olen;
      float* yr = Y + orow * p.ldy;
      const float* rr = R ? R + orow * p.ldr : nullptr;
#pragma unroll
      for (int jn = 0; jn < BN / 8; ++jn) {
        const int n = n0 + jn * 8 + 2 * (lane & 3);
        float v[2] = {acc[mt][4 * jn + 2 * hh], acc[mt][4 * jn + 2 * hh + 1]};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float t = v[e];
          if (n + e < p.N) {
            if (bias) t += bias[n + e];
            if (rr) t += rr[n + e];
            t = conv_act(t, p.act, p.slope);
            v[e] = live ? t : 0.f;
          }
        }
        if (n + 2 <= p.N && ((reinterpret_cast<uintptr_t>(yr + n) & 7) == 0)) {
          *reinterpret_cast<float2*>(yr + n) = make_float2(v[0], v[1]);
        } else {
          if (n < p.N) yr[n] = v[0];
          if (n + 1 < p.N) yr[n + 1] = v[1];
        }
      }
    }
  }
}

template <int BN, int MT>
static int launch_tc(TP& p, cudaStream_t st) {
  constexpr int B_PITCH = BN + 4;
  const int span = (p.off_max - p.off_min) * p.P;
  const long long rows = (long long)MT * 128 + span;
  const long long pitch = ((rows + 7) / 8) * 8 + 4;              // == 4 (mod 8): conflict-free 16-byte panel writes
  // stage shape: KCH 16-byte K-chunks (KC = 4*KCH channels) and TG taps per stage
  auto plan = [&](int kch, int& tg, int& ng) {
    const long long tap_bytes = (long long)kch * B_PITCH * 16;
    tg = (int)max(1LL, min((long long)p.Q, (36 * 1024) / tap_bytes));
    ng = (p.Q + tg - 1) / tg;
    tg = (p.Q + ng - 1) / ng;
    return 2 * (long long)kch * pitch * 16 + 2 * (long long)tg * tap_bytes;
  };
  int KCH = p.C >= 32 ? 8 : (p.C >= 16 ? 4 : 2), TG = 1, NG = 1;
  long long smem = plan(KCH, TG, NG);
  if (smem > 110 * 1024 && KCH == 8) {                            // smaller stages when they fit 110 KB (two CTAs per SM where registers allow)
    int tg2, ng2;
    long long s2 = plan(4, tg2, ng2);
    if (s2 <= 110 * 1024) { KCH = 4; TG = tg2; NG = ng2; smem = s2; }
  }
  if (smem > 200 * 1024 || pitch > 16383) return 1;               // caller falls back to the mma.sync kernel
  p.KCH = KCH; p.TG = TG; p.NG = NG; p.slab_rows = (int)rows; p.a_pitch = (int)pitch;
  auto kern = gconv_tc_kernel<BN, MT>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr_set = true;
  }
  dim3 grid(cdiv((long long)p.J * p.P, MT * 128), cdiv(p.N, BN), p.Z);
  if (grid.x == 0) return EVK_OK;
  if (grid.y > 65535 || grid.z > 65535) return 1;
  kern<<<grid, TC_THREADS, (size_t)smem, st>>>(p);
  return check_launch("gconv_tc_kernel");
}

// c: the launch as evk_gconv_fwd validated it.  Returns 0 on success, < 0 on error, 1 if this launch is not eligible
// (caller uses the mma.sync kernel).
int gconv_tc_try(const ConvP& c, cudaStream_t st) {
  if (c.is != 1 || (c.C % 4) != 0 || c.J <= 0) return 1;
  TP p;
  static_cast<ConvP&>(p) = c;
  const long long npos = (long long)c.J * c.P;
  const bool two = npos >= 4 * 128;                              // two M tiles per CTA: each weight tile is reused twice (flop/byte wins over CTA count)
  const int N = c.N;
  if (N > 64) return two ? launch_tc<128, 2>(p, st) : launch_tc<128, 1>(p, st);
  if (N > 32) return two ? launch_tc<64, 2>(p, st) : launch_tc<64, 1>(p, st);
  if (N > 16) return two ? launch_tc<32, 2>(p, st) : launch_tc<32, 1>(p, st);
  return two ? launch_tc<16, 2>(p, st) : launch_tc<16, 1>(p, st);
}

}  // namespace evk
