// TMA-fed, warp-specialised, persistent wgmma GEMM (sm_90a):   D[M][N] (+)= epi( A[M][K] * B[N][K]^T )
// fp32 storage, TF32 tensor-core math, fp32 accumulation in registers.  Serves every dense contraction without taps:
// nn.Linear / 1x1 conv forward (A = activations rows, B = packed weight [N][C]), their data gradients
// (A = dY rows, B = packed transposed weight [C][N]) and, through evk_gemm_tf32 with split-K, weight gradients on
// pre-transposed operands.  Conv weight gradients run on conv_wgrad_kernel (below), which shares the TMA / mbarrier plumbing.
//
//   warp 0 (one lane)  : TMA producer.  cp.async.bulk.tensor 2-D boxes [128 x 32 fl] (A) and [BN x 32 fl] (B), 128-byte
//                        swizzle, into SA / SB-deep shared-memory rings; full[s] mbarrier with expect_tx.
//   warps 4..11        : two consumer warpgroups.  Warpgroup g owns rows 64 g .. 64 g + 63 of every 128-row block: per
//                        stage 4 x wgmma.m64nBNk8 (K = 8) per block, descriptors advance 32 B inside the 128-byte swizzle
//                        atom.  One wgmma group stays in flight; when the previous group has retired its stages are
//                        released (empty[s], one arrival per consumer warp).  After the last K block of a tile the
//                        warpgroup runs the epilogue from its registers: bias / residual / activation / dropout, 128-byte
//                        row segments to global (split-K: to a per-split partial), while the producer already stages the next
//                        tile.
// CTAs are persistent (one per SM) and walk the tile list n-fastest so that concurrent CTAs share the A row block in L2.
// Out-of-range rows / K tails are zero-filled by TMA, so no shape needs padding.
#include <cuda.h>

#include "wgmma.cuh"

namespace evk {
namespace {

constexpr int BM = 128, BK = 32;                    // 32 floats = one 128-byte swizzle row
constexpr int GT_THREADS = 384;                     // producer warpgroup (warp 0 issues TMA) + two consumer warpgroups
constexpr int CONSUMER_WARPS = 8;

struct GemmP {
  float* d; int ldd;
  const float* bias; const float* res; int ldr;
  int M, N, K, act; float slope;                     // M = output positions per batch item, K = input channels
  int tiles_m, tiles_n, splits, kb_per_split;        // kb = K blocks of 32
  int atomic;                                        // accumulate into d: with d_ssp > 0 each K split stores its partial at
                                                     // d + split * d_ssp (ordered_sum adds them), with d_ssp == 0 (one split) d += result
  long long d_ssp;
  // implicit-GEMM convolution mode (stride 1): Z batch items, Q taps, period P; tap q reads input row pos + off[q]*P
  int Z, Q, P;
  int os, o0;                                        // output position of tile row pos: ((o0 + (pos / P) * os) * P + pos % P)
  int src[EVK_MAX_TAPS];                             // which of the (up to 4) A tensor maps tap q reads (stride phases)
  long long y_sb, r_sb;
  const int* out_len;
  int off[EVK_MAX_TAPS];
  // staging geometry (host-chosen): SA / SB ring depths, a_stage = shared-memory pitch of an A stage (multiple of 1024),
  // a_bytes = bytes the TMA loads of one A stage deliver (expect_tx), slab mode: off_min, span rows after the MT*128-row box
  int SA, SB, a_stage, a_bytes, slab, off_min;
  int fast;                                          // epilogue: every pointer / pitch 16-byte aligned, N % 4 == 0, no atomics, no tanh
  float comp;                                        // accumulator scale compensating the tensor core's operand TRUNCATION (see run_gemm)
  const unsigned long long* drop_rng; unsigned long long drop_sid; float drop_p;   // fused dropout after the activation (0: off)
};

// Fast epilogue rows of one 16 x 32 chunk: this lane owns columns nn .. nn+3 of rows i*4 + r_sub (i = 0..3).  Straight-line
// code: the only conditionals left are single predicated loads / stores.
template <bool RES, bool DROP>
__device__ __forceinline__ void epi_rows_fast(const float* __restrict__ tr, int r_sub, int c4, float4 bv, float* __restrict__ dz,
                                              const float* __restrict__ rz, const size_t (&orow)[4], const bool (&keep)[4],
                                              const bool (&ok)[4], int ldd, int ldr, int nn, float neg, const DropK& dropk,
                                              const float* dbase) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float4 t = *reinterpret_cast<const float4*>(tr + (i * 4 + r_sub) * 36 + c4);
    float* dp = dz + orow[i] * ldd + nn;
    t.x += bv.x; t.y += bv.y; t.z += bv.z; t.w += bv.w;
    if (RES) {
      float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok[i]) rv = *reinterpret_cast<const float4*>(rz + orow[i] * ldr + nn);
      t.x += rv.x; t.y += rv.y; t.z += rv.z; t.w += rv.w;
    }
    t.x = keep[i] ? (t.x > 0.f ? t.x : t.x * neg) : 0.f; t.y = keep[i] ? (t.y > 0.f ? t.y : t.y * neg) : 0.f;
    t.z = keep[i] ? (t.z > 0.f ? t.z : t.z * neg) : 0.f; t.w = keep[i] ? (t.w > 0.f ? t.w : t.w * neg) : 0.f;
    if (DROP) {
      float m[4];
      dropk_scale4(dropk, (unsigned long long)(dp - dbase) >> 2, m);
      t.x *= m[0]; t.y *= m[1]; t.z *= m[2]; t.w *= m[3];
    }
    if (ok[i]) *reinterpret_cast<float4*>(dp) = t;
  }
}

// One 16-row x 32-column chunk of a warp's accumulator, staged row-major in `tr` (pitch 36), to global memory.
// Lane owns columns c4 .. c4+3 of rows i*4 + r_sub.
__device__ __forceinline__ void epi_chunk(const GemmP& p, const float* __restrict__ tr, int lane, int n, float* dz, const float* rz,
                                          const size_t (&orow)[4], const bool (&keep)[4], const bool (&inside)[4], float neg,
                                          const DropK& dropk) {
  const int r_sub = lane >> 3, c4 = (lane & 7) * 4;
  const int nn = n + c4;
  if (p.fast) {
    const bool colok = nn < p.N;                          // N % 4 == 0: the float4 is entirely inside or outside
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias && colok) bv = *reinterpret_cast<const float4*>(p.bias + nn);
    bool ok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) ok[i] = inside[i] && colok;
    if (dropk.thr) {
      if (rz) epi_rows_fast<true, true>(tr, r_sub, c4, bv, dz, rz, orow, keep, ok, p.ldd, p.ldr, nn, neg, dropk, p.d);
      else epi_rows_fast<false, true>(tr, r_sub, c4, bv, dz, rz, orow, keep, ok, p.ldd, p.ldr, nn, neg, dropk, p.d);
    } else if (rz) {
      epi_rows_fast<true, false>(tr, r_sub, c4, bv, dz, rz, orow, keep, ok, p.ldd, p.ldr, nn, neg, dropk, p.d);
    } else {
      epi_rows_fast<false, false>(tr, r_sub, c4, bv, dz, rz, orow, keep, ok, p.ldd, p.ldr, nn, neg, dropk, p.d);
    }
    return;
  }
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool full4 = nn + 4 <= p.N;
  if (p.bias && !p.atomic) {
    if (full4 && ((reinterpret_cast<uintptr_t>(p.bias + nn) & 15) == 0)) bv = *reinterpret_cast<const float4*>(p.bias + nn);
    else { if (nn < p.N) bv.x = p.bias[nn]; if (nn + 1 < p.N) bv.y = p.bias[nn + 1]; if (nn + 2 < p.N) bv.z = p.bias[nn + 2]; if (nn + 3 < p.N) bv.w = p.bias[nn + 3]; }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (!inside[i] || nn >= p.N) continue;
    const float4 tv = *reinterpret_cast<const float4*>(tr + (i * 4 + r_sub) * 36 + c4);
    float t[4] = {tv.x, tv.y, tv.z, tv.w};
    float* dp = dz + orow[i] * p.ldd + nn;
    if (p.atomic) {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (nn + e < p.N) dp[e] = p.d_ssp ? t[e] : dp[e] + t[e];
      continue;
    }
    t[0] += bv.x; t[1] += bv.y; t[2] += bv.z; t[3] += bv.w;
    if (rz) {
      const float* rp = rz + orow[i] * p.ldr + nn;
      if (full4 && ((reinterpret_cast<uintptr_t>(rp) & 15) == 0)) {
        const float4 rv = *reinterpret_cast<const float4*>(rp);
        t[0] += rv.x; t[1] += rv.y; t[2] += rv.z; t[3] += rv.w;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (nn + e < p.N) t[e] += rp[e];
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      t[e] = conv_act(t[e], p.act, p.slope);
      if (!keep[i]) t[e] = 0.f;
    }
    if (dropk.thr) {                                     // group index = offset of the float4 in the output tensor / 4
      float m[4];
      dropk_scale4(dropk, (unsigned long long)(dp - p.d) >> 2, m);
      t[0] *= m[0]; t[1] *= m[1]; t[2] *= m[2]; t[3] *= m[3];
    }
    if (full4 && ((reinterpret_cast<uintptr_t>(dp) & 15) == 0)) {
      *reinterpret_cast<float4*>(dp) = make_float4(t[0], t[1], t[2], t[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (nn + e < p.N) dp[e] = t[e];
    }
  }
}

struct MapB4 { CUtensorMap m[4]; };                  // B: only m[0];  A: one map per stride phase of the input;
                                                     //    slab mode: m[1] = the same tensor with a `span`-row box (the slab tail)
constexpr int MAX_RING = 8;

// One CTA per SM, persistent over the tile list.  Tile = (MT x 128) output rows x BN output channels.
//   MT = 2 : two 128-row blocks share every weight (B) tile -> half the L2->SM weight traffic per flop.
//   slab   : stride-1 tap sums stage ONE input slab of MT*128 + span rows per channel block and run every tap from it
//            (tap q = the A descriptor advanced by (off[q] - off_min) * P rows; see wg_desc_sw128) instead of re-fetching the
//            A box of every tap from L2.
template <int BN, int MT>
__global__ void __launch_bounds__(GT_THREADS, 1) gemm_tma_kernel(const __grid_constant__ MapB4 mapA4,
                                                                 const __grid_constant__ MapB4 mapB4,
                                                                 const __grid_constant__ GemmP p) {
  const CUtensorMap& mapA = mapA4.m[0];
  const CUtensorMap& mapB = mapB4.m[0];
  constexpr int B_BYTES = BN * BK * 4;
  extern __shared__ uint8_t gsm_raw[];
  uint8_t* gsm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gsm_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* gsmB = gsm + (size_t)p.SA * p.a_stage;           // B ring behind the A ring (a_stage is a multiple of 1024)
  __shared__ __align__(8) uint64_t fullA[MAX_RING], emptyA[MAX_RING], fullB[MAX_RING], emptyB[MAX_RING];
  __shared__ __align__(16) float epi_s[CONSUMER_WARPS * 16 * 36];   // per-consumer-warp transpose tile (pitch 36: 128-bit conflict-free)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < MAX_RING; ++i) {
      mbar_init(&fullA[i], 1); mbar_init(&emptyA[i], CONSUMER_WARPS); mbar_init(&fullB[i], 1); mbar_init(&emptyB[i], CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapA4.m[0])));
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapB4.m[0])));
  }
  __syncthreads();

  const int tiles_mn = p.tiles_m * p.tiles_n;
  // tile -> (outer = batch item or K split, m tile, n tile); K iterations = taps x channel blocks (splits > 1 only in plain
  // GEMM mode, Z == Q == 1)
  const int total = tiles_mn * p.splits * p.Z;
  const int kb_total = (p.K + BK - 1) / BK;
  auto k_range = [&](int outer, int& k0, int& k1) {
    if (p.splits > 1) { k0 = outer * p.kb_per_split; k1 = min(kb_total, k0 + p.kb_per_split); }
    else { k0 = 0; k1 = p.Q * kb_total; }
  };
  const int slab = p.slab;

  // Both loops below run once per (tap, channel block) step: ring positions and the (tap, block) decomposition are carried
  // incrementally -- no integer division or modulo by run-time values inside the step loops.
  const int SA = p.SA, SB = p.SB, Q = p.Q;
  if (warp == 0) {
    // The whole warp walks the tile list with warp-uniform state; only the elected lane touches the barriers' tx counts and
    // issues the TMA (a loop under `lane == 0` makes the compiler wrap every TMA issue in a divergence loop).
    int sA = 0, phA = 1, sB = 0, phB = 1;                      // empty barriers: the first pass over a ring passes immediately
    const bool leader = elect_one();
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int outer = tile / tiles_mn, mn = tile - outer * tiles_mn;
      const int tm = mn / p.tiles_n, tn = mn - tm * p.tiles_n;
      const int z = p.splits > 1 ? 0 : outer;
      auto next_a = [&]() -> uint8_t* {
        mbar_wait(&emptyA[sA], phA);
        if (leader) mbar_expect_tx(&fullA[sA], (uint32_t)p.a_bytes);
        return gsm + (size_t)sA * p.a_stage;
      };
      auto done_a = [&]() { if (++sA == SA) { sA = 0; phA ^= 1; } };
      auto next_b = [&]() -> uint8_t* {
        mbar_wait(&emptyB[sB], phB);
        if (leader) mbar_expect_tx(&fullB[sB], B_BYTES);
        return gsmB + (size_t)sB * B_BYTES;
      };
      auto done_b = [&]() { if (++sB == SB) { sB = 0; phB ^= 1; } };
      if (slab) {
        const int row0 = tm * (MT * BM) + p.off_min * p.P;
        for (int kb = 0; kb < kb_total; ++kb) {
          uint8_t* sa = next_a();
          if (leader) tma_load_3d(sa, &mapA, kb * BK, row0, z, &fullA[sA]);
          if (leader) tma_load_3d(sa + MT * BM * BK * 4, &mapA4.m[1], kb * BK, row0 + MT * BM, z, &fullA[sA]);
          done_a();
          for (int q = 0; q < Q; ++q) {
            uint8_t* sb = next_b();
            if (leader) tma_load_3d(sb, &mapB, kb * BK, tn * BN, q, &fullB[sB]);
            done_b();
          }
        }
      } else if (p.splits == 1) {
        for (int q = 0; q < Q; ++q) {
          const CUtensorMap* am = &mapA4.m[p.src[q]];
          const int arow = tm * (MT * BM) + p.off[q] * p.P;
          for (int kb = 0; kb < kb_total; ++kb) {
            uint8_t* sa = next_a();
            if (leader) tma_load_3d(sa, am, kb * BK, arow, z, &fullA[sA]);
            done_a();
            uint8_t* sb = next_b();
            if (leader) tma_load_3d(sb, &mapB, kb * BK, tn * BN, q, &fullB[sB]);
            done_b();
          }
        }
      } else {                                                 // split-K plain GEMM (Z == Q == 1)
        int k0, k1;
        k_range(outer, k0, k1);
        for (int kb = k0; kb < k1; ++kb) {
          uint8_t* sa = next_a();
          if (leader) tma_load_3d(sa, &mapA, kb * BK, tm * (MT * BM), 0, &fullA[sA]);
          done_a();
          uint8_t* sb = next_b();
          if (leader) tma_load_3d(sb, &mapB, kb * BK, tn * BN, 0, &fullB[sB]);
          done_b();
        }
      }
    }
  } else if (warp >= 4) {
    const int cw = warp - 4;                                   // consumer warp 0..7
    const int wg = cw >> 2, wq = cw & 3;                       // warpgroup (64-row half of a 128-row block), warp in it (16 rows)
    float* tr = epi_s + cw * (16 * 36);
    const float comp = p.comp;
    const DropK dropk = dropk_make(p.drop_rng, p.drop_sid, p.drop_p);
    const float neg = p.act == EVK_ACT_LRELU ? p.slope : (p.act == EVK_ACT_RELU ? 0.f : 1.f);   // fast path: x > 0 ? x : x * neg
    int sA = 0, phA = 0, sB = 0, phB = 0;
    const uint32_t a_ring = smem_u32(gsm) + (uint32_t)(wg * 64 * BK * 4), b_ring = smem_u32(gsmB);
    float acc[MT][BN / 2];
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      // ---- main loop: one wgmma group per step in flight; the stages of the step before it are released once it retires
      int relA = -1, relB = -1;
      uint32_t accum = 0;
      auto step = [&](uint32_t a_off) {
        mbar_wait(&fullB[sB], phB);
        const int ra = relA;
        relA = -1;
        const uint32_t a_addr = a_ring + (uint32_t)sA * (uint32_t)p.a_stage + a_off;
        const uint64_t db = wg_desc_sw128(b_ring + (uint32_t)sB * B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const uint64_t da = wg_desc_sw128(a_addr + (uint32_t)(mt * BM * BK * 4));
#pragma unroll
          for (int k = 0; k < BK / 8; ++k) wgmma_tf32<BN>(acc[mt], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), accum | (uint32_t)k);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (lane == 0) {
          if (relB >= 0) mbar_arrive(&emptyB[relB]);
          if (ra >= 0) mbar_arrive(&emptyA[ra]);
        }
        relB = sB;
        accum = 1;
        if (++sB == SB) { sB = 0; phB ^= 1; }
      };
      auto wait_a = [&]() { mbar_wait(&fullA[sA], phA); };
      auto free_a = [&]() { relA = sA; if (++sA == SA) { sA = 0; phA ^= 1; } };
      if (slab) {
        for (int kb = 0; kb < kb_total; ++kb) {
          wait_a();
          for (int q = 0; q < Q; ++q) step((uint32_t)((p.off[q] - p.off_min) * p.P) * (BK * 4));
          free_a();
        }
      } else {
        int k0, k1;
        k_range(tile / tiles_mn, k0, k1);
        for (int ki = k0; ki < k1; ++ki) {
          wait_a();
          step(0);
          free_a();
        }
      }
      wgmma_wait<0>();
      if (lane == 0) {
        if (relB >= 0) mbar_arrive(&emptyB[relB]);
        if (relA >= 0) mbar_arrive(&emptyA[relA]);
      }
      if (!accum) {                                            // empty K range (cannot happen for a listed tile): write zeros
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[mt][i] = 0.f;
      }

      // ---- epilogue from registers
      const int outer = tile / tiles_mn, mn = tile - outer * tiles_mn;
      const int tm = mn / p.tiles_n, tn = mn - tm * p.tiles_n;
      const int z = p.splits > 1 ? 0 : outer;
      float* dz = p.d + (size_t)z * p.y_sb;
      if (p.atomic) dz += (size_t)outer * p.d_ssp;
      const float* rz = p.res ? p.res + (size_t)z * p.r_sb : nullptr;
      const int olen = p.out_len ? p.out_len[z] : 0x7fffffff;
      const int r_sub = lane >> 3;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int row_base = tm * (MT * BM) + mt * BM + wg * 64 + wq * 16;
        if (row_base >= p.M) continue;                           // warp-uniform: nothing of this warp's rows is inside the problem
        // this lane's 4 rows (rl = i*4 + r_sub): output row index and length-mask flag, once per block
        size_t orow[4];
        bool keep[4], inside[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = row_base + i * 4 + r_sub;
          inside[i] = row < p.M;
          int jo;
          if (p.P == 1) { jo = p.o0 + row * p.os; orow[i] = (size_t)jo; }
          else { const int jq = row / p.P; jo = p.o0 + jq * p.os; orow[i] = (size_t)jo * p.P + (row - jq * p.P); }
          keep[i] = jo < olen;
        }
#pragma unroll
        for (int c = 0; c < BN / 32; ++c) {
          const int n = tn * BN + c * 32;
          if (n >= p.N) break;                                   // warp-uniform
          // fragment -> row-major 16 x 32 tile: d[4j + 2h + e] = (row lane/4 + 8h, column 8j + 2(lane%4) + e)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int j = c * 4 + jj;
              *reinterpret_cast<float2*>(tr + ((lane >> 2) + 8 * h) * 36 + jj * 8 + 2 * (lane & 3)) =
                  make_float2(acc[mt][4 * j + 2 * h] * comp, acc[mt][4 * j + 2 * h + 1] * comp);
            }
          __syncwarp();
          epi_chunk(p, tr, lane, n, dz, rz, orow, keep, inside, neg, dropk);
          __syncwarp();
        }
      }
    }
  }
}

// [outer][rows][K] fp32 (row pitch ld, outer pitch sb, in floats): box = [1][box_rows][32 floats], 128-byte swizzle.
// Rows outside [0, rows) -- negative tap offsets included -- and channels past K are zero-filled by the TMA unit.
bool make_map(CUtensorMap* m, const float* base, long long outer, long long sb, long long rows, long long K, long long ld, int box_rows) {
  if (K <= 0 || rows <= 0 || outer <= 0 || K > 0xffffffffll || rows > 0xffffffffll) return false;
  EncodeFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)outer};
  cuuint64_t gstr[2] = {(cuuint64_t)ld * 4, (cuuint64_t)(outer > 1 ? sb : rows * ld) * 4};
  cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int g_sm_count = 0;
int sm_count() {
  if (!g_sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_sm_count;
}
int g_opt_slab = 1, g_opt_mt2 = 1;          // A/B switches (evk_set_tma_options)
// The tensor core reads fp32 operands as TF32 by DROPPING the low 13 mantissa bits (truncation towards zero): every product
// is biased by -2^-11 * E[1/m] = -3.5e-4 relative per truncated operand (m = mantissa in [1,2), log-uniform).  Weights are
// rounded to nearest once when they are packed, activations arrive raw through TMA.  The bias is systematic -- it adds up
// along a 24-layer residual stream and shows in LayerNorm's 1/sigma (measured on the 24-layer GPT: gradient norms drift by
// +1 % over 16 layers, d alpha off by 3x the noise bound) -- so the epilogue multiplies the accumulator by
// (1 + 3.52e-4)^(number of raw operands).  The variance of the per-element error is the same as round-to-nearest's.
float g_trunc_comp = 3.52e-4f;

struct Operands {
  const float* A; int lda; long long a_sb, a_rows;     // activations: [Z][a_rows][K]
  const float* B; int ldb; long long b_sq;             // weights:     [Q][N][K]
  int a_phases; long long a_ps;                        // stride phases of the input and their pitch
  int raw_operands;                                    // how many of the two operands are un-rounded fp32 (truncated by the MMA)
};

constexpr int SMEM_BUDGET = 200 * 1024;               // + 1 KB alignment + 18.4 KB static epilogue tiles + barriers <= 227 KB

template <int BN, int MT>
int launch_gemm(const Operands& o, GemmP& p, int splits, cudaStream_t st) {
  constexpr int B_BYTES = BN * BK * 4;
  MapB4 ma, mb;
  p.slab = 0;
  int span = 0;
  if (g_opt_slab && o.a_phases == 1 && p.Q >= 2 && splits <= 1) {
    int mn = p.off[0], mx = p.off[0];
    for (int i = 1; i < p.Q; ++i) { mn = min(mn, p.off[i]); mx = max(mx, p.off[i]); }
    span = (mx - mn) * p.P;
    const long long a_stage = ((long long)(MT * BM + span + 7) / 8 * 8) * BK * 4;
    if (span >= 1 && span <= 256 && (SMEM_BUDGET - 2 * a_stage) / B_BYTES >= 3) {
      p.slab = 1; p.off_min = mn; p.SA = 2; p.a_stage = (int)a_stage; p.a_bytes = (MT * BM + span) * BK * 4;
      { const long long nb = (SMEM_BUDGET - 2 * a_stage) / B_BYTES; p.SB = (int)(nb < MAX_RING ? nb : MAX_RING); }
    }
  }
  if (!p.slab) {
    p.a_stage = p.a_bytes = MT * BM * BK * 4;
    p.SA = p.SB = min(MAX_RING, SMEM_BUDGET / (p.a_stage + B_BYTES));
  }
  for (int ph = 0; ph < 4; ++ph) {
    if (ph < o.a_phases) { if (!make_map(&ma.m[ph], o.A + ph * o.a_ps, p.Z, o.a_sb, o.a_rows, p.K, o.lda, MT * BM)) return 1; }
    else ma.m[ph] = ma.m[0];
  }
  if (p.slab && !make_map(&ma.m[1], o.A, p.Z, o.a_sb, o.a_rows, p.K, o.lda, span)) return 1;
  if (!make_map(&mb.m[0], o.B, p.Q, o.b_sq, p.N, p.K, o.ldb, BN)) return 1;
  mb.m[1] = mb.m[2] = mb.m[3] = mb.m[0];
  const size_t SMEM = (size_t)p.SA * p.a_stage + (size_t)p.SB * B_BYTES + 1024;
  auto kern = gemm_tma_kernel<BN, MT>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET + 1024) != cudaSuccess) return 1;
    attr_set = true;
  }
  p.comp = 1.f;
  for (int i = 0; i < o.raw_operands; ++i) p.comp *= 1.f + g_trunc_comp;
  {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const bool act_ok = p.act == EVK_ACT_NONE || p.act == EVK_ACT_LRELU || p.act == EVK_ACT_RELU;
    p.fast = (act_ok && !p.atomic && (p.N % 4) == 0 && (p.ldd % 4) == 0 && (p.y_sb % 4) == 0 && al16(p.d) && (!p.bias || al16(p.bias)) &&
              (!p.res || (al16(p.res) && (p.ldr % 4) == 0 && (p.r_sb % 4) == 0))) ? 1 : 0;
  }
  p.tiles_m = cdiv(p.M, MT * BM);
  p.tiles_n = cdiv(p.N, BN);
  const int kb_total = cdiv(p.K, BK);
  splits = max(1, min(splits, kb_total));
  p.kb_per_split = cdiv(kb_total, splits);
  p.splits = cdiv(kb_total, p.kb_per_split);
  // split-K partials: [split][M][N] in scratch (bounded: fewer splits when a large output would not fit)
  const long long outq = (long long)p.M * p.N;
  float* dst = p.d;
  const long long dst_ld = p.ldd;
  Scratch part_buf(0, st);
  if (p.atomic) {
    constexpr long long PART_CAP = 32ll << 20;
    if ((long long)p.splits * outq > PART_CAP) {
      splits = (int)max(1ll, PART_CAP / outq);
      p.kb_per_split = cdiv(kb_total, splits);
      p.splits = cdiv(kb_total, p.kb_per_split);
    }
    p.d_ssp = 0;
    if (p.splits > 1) {                                   // one split: every element has one writer, which adds in place
      part_buf.alloc((long long)p.splits * outq);
      p.d = part_buf.p;
      EVK_REQUIRE(p.d, EVK_ERR_CUDA, "gemm_tma: scratch allocation failed");
      p.ldd = p.N; p.d_ssp = outq;
    }
  }
  const long long total = (long long)p.tiles_m * p.tiles_n * p.splits * p.Z;
  if (total > 0x7fffffff) return 1;
  if (total <= 0) return EVK_OK;
  const int grid = (int)(total < (long long)g_sm_count ? total : (long long)g_sm_count);
  kern<<<grid, GT_THREADS, SMEM, st>>>(ma, mb, p);
  if (int rc = check_launch("gemm_tma_kernel")) return rc;
  return (p.atomic && p.d_ssp) ? ordered_sum(p.d, p.splits, outq, 1, p.M, p.N, dst, 0, dst_ld, st) : EVK_OK;
}

// MT = 2 halves the weight-tile traffic per flop but doubles the tile: take it when the wave quantisation of the persistent
// grid does not eat the gain (cost in units of 128-row tile-times; 0.65 = relative cost of a row in a 256-row tile).  Only
// the 32-channel layers use it: they are bound by operand traffic, the wider ones by the tensor core.
template <int BN>
int launch_bn(const Operands& o, GemmP& p, int splits, cudaStream_t st) {
  sm_count();
  if constexpr (BN == 32) {
    if (g_opt_mt2 && splits <= 1 && p.M >= 2 * BM) {
      const long long per = (long long)cdiv(p.N, BN) * p.Z;
      const long long t1 = per * cdiv(p.M, BM), t2 = per * cdiv(p.M, 2 * BM);
      const double c1 = (double)cdiv(t1, g_sm_count), c2 = (double)cdiv(t2, g_sm_count) * 2.0 * 0.65;
      if (c2 < c1) return launch_gemm<BN, 2>(o, p, splits, st);
    }
  }
  return launch_gemm<BN, 1>(o, p, splits, st);
}

// Tile width: the widest that the output channels fill.  128 is the cap: the 64 x 128 fp32 accumulator of a consumer
// warpgroup already takes 64 registers per thread, and a 128-row x 128-column tile reads each staged A byte for 128 columns.
int run_gemm(const Operands& o, GemmP& p, int splits, cudaStream_t st) {
  if (p.N > 64) return launch_bn<128>(o, p, splits, st);
  if (p.N > 32) return launch_bn<64>(o, p, splits, st);
  return launch_bn<32>(o, p, splits, st);
}


// ---- conv weight gradient: dW[q][n][c] = sum_b sum_pos dY[b][pos][n] * X[b][pos + off[q] * P][c] -----------------------
// The GEMM runs transposed, D[(q, c)][n]: the M rows are (tap, input channel) pairs, so one output tile holds 128 / C taps
// of a narrow layer (4 at 32 channels, 2 at 64) and every tap of the tile shares the staged dY block.  K = positions.
//   X side (A, from registers): per K block of 32 positions the producer stages, for each 32-row quarter of the tile,
//     the channels-last box X[b][t0 + shift .. + 31][c0 .. c0 + 31] (128-byte swizzle).  The tap shift is the box's row
//     coordinate (rows outside the input = the conv padding, zero-filled by the copy engine), so X is read in the layout
//     the forward left it -- no transposed or delayed copies.  The consumer threads load their A fragments from that
//     box with ordinary shared-memory loads (TF32 wgmma takes A from registers in any source layout).
//   dY side (B, from shared memory): the K-major box dyt[b][n0 .. n0 + BN - 1][t0 .. t0 + 31] of the transposed output
//     gradient that evk_dy_prep writes in its pass over dY (positions past the output are zero-filled).
// Work item = (K split, m tile, n tile), n fastest; K iterations = batch items x 32-position blocks.  Splits store their
// partials, which ordered_sum adds in split order, so the result does not depend on the schedule.
struct WgradP {
  float* d; int ldd; long long d_sq, d_ssp;           // output (pitch ldd, tap pitch d_sq); d_ssp > 0: split partials, else d += D
  int N, C, Cp, nq, P;                                // Cp = C rounded up to 32: tile row r = q * Cp + c
  int kbs, kb_total, tiles_m, tiles_n, splits, kb_per_split, ring;
  int off[EVK_MAX_TAPS];
  float comp;
};

constexpr int WG_A_BYTES = BM * BK * 4;               // four 32 x 32 X boxes

template <int BN>
__global__ void __launch_bounds__(GT_THREADS, 1) conv_wgrad_kernel(const __grid_constant__ CUtensorMap mapX,
                                                                   const __grid_constant__ CUtensorMap mapD,
                                                                   const __grid_constant__ WgradP p) {
  constexpr int STAGE = WG_A_BYTES + BN * BK * 4;
  extern __shared__ uint8_t gsm_raw[];
  uint8_t* gsm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gsm_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full[MAX_RING], empty[MAX_RING];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < MAX_RING; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;\n");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapX)));
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(&mapD)));
  }
  __syncthreads();
  const int tiles_mn = p.tiles_m * p.tiles_n, total = tiles_mn * p.splits, ring = p.ring;

  if (warp == 0) {
    int s = 0, ph = 1;
    const bool leader = elect_one();
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int sp = tile / tiles_mn, mn = tile - sp * tiles_mn;
      const int tm = mn / p.tiles_n, tn = mn - tm * p.tiles_n;
      const int k0 = sp * p.kb_per_split, k1 = min(p.kb_total, k0 + p.kb_per_split);
      int c0[4], sh[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {                            // quarter j of the tile = 32 channels of one tap
        const int g = tm * 4 + j, per = p.Cp / 32;
        const int q = min(g / per, p.nq - 1);                  // past the last tap: loaded, never written
        c0[j] = (g - (g / per) * per) * 32;
        sh[j] = p.off[q] * p.P;
      }
      int b = k0 / p.kbs, kk = k0 - b * p.kbs;
      for (int ki = k0; ki < k1; ++ki) {
        mbar_wait(&empty[s], ph);
        if (leader) {
          uint8_t* st = gsm + (size_t)s * STAGE;
          mbar_expect_tx(&full[s], STAGE);
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_3d(st + j * (BK * BK * 4), &mapX, c0[j], kk * BK + sh[j], b, &full[s]);
          tma_load_3d(st + WG_A_BYTES, &mapD, kk * BK, tn * BN, b, &full[s]);
        }
        if (++s == ring) { s = 0; ph ^= 1; }
        if (++kk == p.kbs) { kk = 0; ++b; }
      }
    }
  } else if (warp >= 4) {
    const int cw = warp - 4, wg = cw >> 2, wq = cw & 3;
    const int r0 = wg * 64 + wq * 16 + (lane >> 2);            // this thread's tile rows r0 and r0 + 8: quarter r0 / 32
    // byte offsets of A(r0 + 8 e, k = lane % 4 + 4 h) in the swizzled box of quarter r0 / 32:
    // position row k * 128, 16-byte chunk (channel / 4) ^ (k % 8); K step kstep adds 8 positions = 1024 bytes
    uint32_t aoff[2][2];
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cl = (r0 & 31) + 8 * e, k = (lane & 3) + 4 * h;
        aoff[e][h] = (uint32_t)((r0 >> 5) * (BK * BK * 4) + k * 128 + ((((cl >> 2) ^ k) & 7) << 4) + (cl & 3) * 4);
      }
    const uint32_t ring_base = smem_u32(gsm);
    int s = 0, ph = 0;
    float acc[BN / 2];
    float ra[BK / 8][4];
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int sp = tile / tiles_mn, mn = tile - sp * tiles_mn;
      const int tm = mn / p.tiles_n, tn = mn - tm * p.tiles_n;
      const int k0 = sp * p.kb_per_split, k1 = min(p.kb_total, k0 + p.kb_per_split);
      int rel = -1;
      uint32_t accum = 0;
      // One K block: retire the previous block's wgmma group (it read the A registers and the previous stage), load this
      // block's A fragments, issue its four k8 steps.  The fragment loads overlap the TMA of the stages ahead.
      for (int ki = k0; ki < k1; ++ki) {
        mbar_wait(&full[s], ph);
        wgmma_wait<0>();
        if (lane == 0 && rel >= 0) mbar_arrive(&empty[rel]);
        const uint32_t sa = ring_base + (uint32_t)s * STAGE;
#pragma unroll
        for (int k = 0; k < BK / 8; ++k)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              uint32_t v;
              asm volatile("ld.shared.b32 %0, [%1];\n" : "=r"(v) : "r"(sa + aoff[e][h] + k * 1024));
              ra[k][2 * h + e] = __uint_as_float(v & 0xffffe000u);    // TF32 by truncation, as the tensor core reads
            }                                                         // a shared-memory operand
        wgmma_fence();
        const uint64_t db = wg_desc_sw128(sa + WG_A_BYTES);
#pragma unroll
        for (int k = 0; k < BK / 8; ++k) wgmma_tf32_rs<BN>(acc, ra[k], db + (uint64_t)(k * 2), accum | (uint32_t)k);
        wgmma_commit();
        rel = s;
        accum = 1;
        if (++s == ring) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0 && rel >= 0) mbar_arrive(&empty[rel]);
      if (!accum) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      }
      // epilogue: D[(q, c)][n] -> dW[q][n][c]; acc[4 j + 2 h + x] = (row r0 + 8 h, column 8 j + 2 (lane % 4) + x)
      float* dz = p.d + (size_t)sp * p.d_ssp;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = tm * BM + r0 + 8 * h, q = row / p.Cp, c = row - q * p.Cp;
        if (q >= p.nq || c >= p.C) continue;
        float* base = dz + (size_t)q * p.d_sq + c;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int x = 0; x < 2; ++x) {
            const int n = tn * BN + 8 * j + 2 * (lane & 3) + x;
            if (n >= p.N) continue;
            float* dp = base + (size_t)n * p.ldd;
            const float v = acc[4 * j + 2 * h + x] * p.comp;
            *dp = p.d_ssp ? v : *dp + v;
          }
      }
    }
  }
}

template <int BN>
int launch_wgrad(const CUtensorMap& mx, const float* dyt, int ld_dy, long long dy_sb, int B, int out_rows, WgradP& p, int splits,
                 cudaStream_t st) {
  constexpr int STAGE = WG_A_BYTES + BN * BK * 4;
  CUtensorMap md;
  if (!make_map(&md, dyt, B, dy_sb, p.N, out_rows, ld_dy, BN)) return 1;
  sm_count();
  p.ring = min(MAX_RING, SMEM_BUDGET / STAGE);
  p.tiles_m = cdiv(p.nq * p.Cp, BM);
  p.tiles_n = cdiv(p.N, BN);
  p.kbs = cdiv(out_rows, BK);
  p.kb_total = B * p.kbs;
  p.comp = (1.f + g_trunc_comp) * (1.f + g_trunc_comp);     // both operands are raw activations / gradients
  // split-K partials [split][nq][N][C] in scratch (bounded: fewer splits when a large output would not fit)
  const long long outq = (long long)p.nq * p.N * p.C;
  constexpr long long PART_CAP = 32ll << 20;
  splits = max(1, min(splits, p.kb_total));
  p.kb_per_split = cdiv(p.kb_total, splits);
  p.splits = cdiv(p.kb_total, p.kb_per_split);
  if ((long long)p.splits * outq > PART_CAP) {
    splits = (int)max(1ll, PART_CAP / outq);
    p.kb_per_split = cdiv(p.kb_total, splits);
    p.splits = cdiv(p.kb_total, p.kb_per_split);
  }
  float* dst = p.d;
  const long long dst_sq = p.d_sq, dst_ld = p.ldd;
  Scratch part_buf(0, st);
  p.d_ssp = 0;
  if (p.splits > 1) {                                     // one split: every element has one writer, which adds in place
    part_buf.alloc((long long)p.splits * outq);
    EVK_REQUIRE(part_buf.p, EVK_ERR_CUDA, "conv_wgrad_tma: scratch allocation failed");
    p.d = part_buf.p; p.ldd = p.C; p.d_sq = (long long)p.N * p.C; p.d_ssp = outq;
  }
  const long long total = (long long)p.tiles_m * p.tiles_n * p.splits;
  if (total > 0x7fffffff) return 1;
  const size_t SMEM = (size_t)p.ring * STAGE + 1024;
  auto kern = conv_wgrad_kernel<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET + 1024) != cudaSuccess) return 1;
    attr_set = true;
  }
  kern<<<(int)min(total, (long long)g_sm_count), GT_THREADS, SMEM, st>>>(mx, md, p);
  if (int rc = check_launch("conv_wgrad_kernel")) return rc;
  return p.d_ssp ? ordered_sum(p.d, p.splits, outq, p.nq, p.N, p.C, dst, dst_sq, dst_ld, st) : EVK_OK;
}

}  // namespace

int g_backend_tma = 1;

// Fills o and p for the launch d: returns 0, or 1 if it is not eligible.  phases > 1: d->x points at `phases` stride-phase
// copies of the input (pitch x_ps floats, see split_phases) and tap q reads copy src[q] with row shift off[q] -- a strided
// conv expressed as a stride-1 multi-source tap sum.
static int gemm_tma_plan(const evk_gconv_desc* d, int phases, long long x_ps, const int* src, Operands& o, GemmP& p) {
  if (!g_backend_tma) return 1;
  if (d->is != 1 || d->os < 1 || d->o0 < 0 || d->H != 1 || d->Q < 1 || d->Q > EVK_MAX_TAPS || phases < 1 || phases > 4) return 1;
  if (d->in_len) return 1;                                  // ragged inputs are masked at staging time by the tap kernel
  if ((d->C % 4) || (d->ldx % 4) || (d->ldw % 4) || (d->ldy % 4) || (d->res && (d->ldr % 4))) return 1;
  if (((uintptr_t)d->x | (uintptr_t)d->w | (uintptr_t)d->y) & 15) return 1;
  if ((d->x_sb % 4) || (d->w_sq % 4) || (x_ps % 4) || (d->Z > 1 && d->w_sb != 0) || d->w_sq < 0 || d->x_sb < 0) return 1;
  const long long npos = (long long)d->J * d->P, in_rows = (long long)d->Tin * d->P;
  p = GemmP{};
  p.d = d->y; p.ldd = d->ldy; p.bias = d->bias; p.res = d->res; p.ldr = d->ldr;
  p.N = d->N; p.K = d->C; p.act = d->act; p.slope = d->slope; p.atomic = 0;
  p.Q = d->Q; p.P = d->P; p.out_len = d->out_len; p.os = d->os; p.o0 = d->o0;
  p.drop_rng = reinterpret_cast<const unsigned long long*>(d->drop_rng); p.drop_sid = d->drop_sid; p.drop_p = d->drop_rng ? d->drop_p : 0.f;
  if (p.drop_p > 0.f && ((d->N % 4) || (d->ldy % 4) || (d->y_sb % 4))) return 1;     // the mask is keyed by float4 groups of the output
  for (int i = 0; i < EVK_MAX_TAPS; ++i) {
    p.off[i] = i < d->Q ? d->off[i] : 0;
    p.src[i] = (src && i < d->Q) ? src[i] : 0;
    if (p.src[i] < 0 || p.src[i] >= phases) return 1;
  }
  o = Operands{};
  o.B = d->w; o.ldb = d->ldw; o.b_sq = d->w_sq; o.a_phases = phases; o.a_ps = x_ps;
  o.raw_operands = 1;                                       // A = activations (raw fp32), B = packed weights (already TF32, rounded to nearest)
  const bool flat = phases == 1 && d->Q == 1 && d->off[0] == 0 && d->P == 1 && !d->out_len && d->J == d->Tin && d->os == 1 && d->o0 == 0 &&
                    (d->Z == 1 || (d->x_sb == in_rows * d->ldx && d->y_sb == npos * d->ldy && (!d->res || d->r_sb == npos * d->ldr)));
  if (flat) {                                               // Linear / 1x1 conv: batch folds into the row dimension
    const long long rows = (long long)d->Z * npos;
    if (rows < 512 || d->C < 64 || d->N < 64 || rows > 0x7fffffff) return 1;
    p.M = (int)rows; p.Z = 1; p.y_sb = 0; p.r_sb = 0;
    o.A = d->x; o.lda = d->ldx; o.a_sb = 0; o.a_rows = rows;
  } else {                                                  // stride-1 tap sum: one TMA box per (tap, channel block), OOB rows = padding
    // 16-channel layers stay on gconv_tc_kernel: routed here, half of every 32-float K box would be out of range
    if (npos < 64 || (long long)d->Z * npos < 1024 || d->C < 32 || d->N < 32 || npos > 0x7fffffff) return 1;
    p.M = (int)npos; p.Z = d->Z; p.y_sb = d->y_sb; p.r_sb = d->r_sb;
    o.A = d->x; o.lda = d->ldx; o.a_sb = d->x_sb; o.a_rows = in_rows;
  }
  return 0;
}

// returns 0 on success, < 0 on error, 1 if this launch is not eligible (caller falls through to gconv_tc / mma.sync)
int gemm_tma_try(const evk_gconv_desc* d, cudaStream_t st) {
  Operands o; GemmP p;
  return gemm_tma_plan(d, 1, 0, nullptr, o, p) ? 1 : run_gemm(o, p, 1, st);
}

// The stride phases of a conv input: tap offset u reads phase copy u mod s at row shift floor(u / s).
static void phase_of(int u, int s, int& copy, int& shift) {
  copy = ((u % s) + s) % s;
  shift = (u - copy) / s;
}

// stride-phase split: xs[rho][b][j*P + w][c] = x[b][(j*s + rho)*P + w][c] (zero when j*s + rho >= T), j < Jp
__global__ void phase_split_kernel(const float* __restrict__ x, int ldx, long long x_sb, float* __restrict__ xs, long long xs_ps,
                                   int B, int T, int P, int C, int s, int Jp) {
  const int c4n = C / 4;
  const long long n = (long long)s * B * Jp * P * c4n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c4 = (int)(i % c4n);
    long long r = i / c4n;
    int w = (int)(r % P); r /= P;
    int j = (int)(r % Jp); r /= Jp;
    int b = (int)(r % B);
    int rho = (int)(r / B);
    const int t = j * s + rho;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < T) v = *reinterpret_cast<const float4*>(x + b * x_sb + ((long long)t * P + w) * ldx + c4 * 4);
    *reinterpret_cast<float4*>(xs + rho * xs_ps + (((long long)b * Jp + j) * P + w) * C + c4 * 4) = v;
  }
}

// d's input split into its `is` stride phases in scratch: copies x_ps floats apart, each [Z][ceil(Tin / is) * P][C]
static int split_phases(const evk_gconv_desc* d, Scratch& xs, long long& x_ps, cudaStream_t st) {
  const int Jp = cdiv(d->Tin, d->is);
  x_ps = (long long)d->Z * Jp * d->P * d->C;
  xs.alloc(d->is * x_ps);
  EVK_REQUIRE(xs.p, EVK_ERR_CUDA, "gconv: scratch allocation for the stride phases failed");
  const int blocks = min(cdiv(d->is * x_ps / 4, 256), kNumSMs * 32);          // grid-stride, a few waves of the SMs
  phase_split_kernel<<<blocks, 256, 0, st>>>(d->x, d->ldx, d->x_sb, xs.p, x_ps, d->Z, d->Tin, d->P, d->C, d->is, Jp);
  return check_launch("phase_split");
}

// evk_gconv_fwd's route 1 for a tileable launch; returns 1 when it does not apply.  All of its rule (here and in gemm_tma_plan:
// H == 1, no in_len, C % 4 == 0, C, N >= 32, J*P >= 64) is checked before the input is split.
int gemm_tma_phased(const evk_gconv_desc* d, cudaStream_t st) {
  const int s = d->is, C = d->C;
  if (s < 2 || s > 4 || d->no_phase_split || (long long)d->Z * d->J * d->P < 2048) return 1;
  evk_gconv_desc e = *d;                                  // the stride-1 tap sum over the phase copies (x set after the split)
  e.ldx = C; e.Tin = cdiv(d->Tin, s); e.x_sb = (long long)e.Tin * d->P * C; e.is = 1;
  int src[EVK_MAX_TAPS];
  for (int q = 0; q < d->Q; ++q) phase_of(d->off[q], s, src[q], e.off[q]);
  Operands o; GemmP p;
  if (gemm_tma_plan(&e, s, (long long)d->Z * e.x_sb, src, o, p)) return 1;
  Scratch xs(0, st);
  long long x_ps;
  if (int rc = split_phases(d, xs, x_ps, st)) return rc;
  o.A = xs.p;
  return run_gemm(o, p, 1, st);
}

// Conv weight gradient on conv_wgrad_kernel (evk_gconv_wgrad's route 1):
//   dW[q][n][c] += sum_b sum_pos dY[b][pos][n] * X[b][pos + off[q]*P][c]
// X is read channels-last as the forward left it (the tap shift is a TMA row coordinate; out-of-range rows = the conv
// padding, zero-filled by the copy engine), dY through dyt [B][N][ld_dyt], its transpose.  The tile rows are (tap, input
// channel) pairs, so the taps of a narrow layer share each staged dY block.  A strided conv is first split into `stride`
// phase copies of X (as in the forward): the taps of one phase form a stride-1 problem on that copy.
int conv_wgrad_tma(const evk_gconv_desc* d, const float* dyt, int ld_dyt, cudaStream_t st) {
  const int s = d->is, B = d->Z, P = d->P, C = d->C, N = d->N, out_rows = d->J * P;
  const long long dy_sb = (long long)N * ld_dyt;
  EVK_REQUIRE((ld_dyt % 4) == 0 && ld_dyt >= out_rows && ((uintptr_t)dyt & 15) == 0, EVK_ERR_ARG,
              "gconv_wgrad: dyt must be 16-byte aligned with a pitch >= J*P that is a multiple of 4 floats");
  const float* x = d->x;
  int ldx = d->ldx, in_rows = d->Tin * P;
  long long x_sb = d->x_sb, x_ps = 0;
  Scratch xs(0, st);
  if (s > 1) {
    if (int rc = split_phases(d, xs, x_ps, st)) return rc;
    x = xs.p; ldx = C; in_rows = cdiv(d->Tin, s) * P; x_sb = (long long)in_rows * C;
  }
  for (int rho = 0; rho < s; ++rho) {
    WgradP p{};
    int qs[EVK_MAX_TAPS], nq = 0;
    for (int q = 0; q < d->Q; ++q) {
      int copy, shift;
      phase_of(d->off[q], s, copy, shift);
      if (copy == rho) { qs[nq] = q; p.off[nq++] = shift; }
    }
    if (!nq) continue;
    CUtensorMap mx;
    EVK_REQUIRE(make_map(&mx, x + rho * x_ps, B, x_sb, in_rows, C, ldx, BK), EVK_ERR_UNSUPPORTED,
                "gconv_wgrad: cuTensorMapEncodeTiled unavailable or rejected the operand");
    p.d = d->w + qs[0] * d->w_sq; p.ldd = d->ldw; p.d_sq = (nq > 1 ? qs[1] - qs[0] : 1) * d->w_sq;
    p.N = N; p.C = C; p.Cp = cdiv(C, 32) * 32; p.nq = nq; p.P = P;
    // the split count fixes how the K sums are grouped, and so the bits of dW: it depends on the layer shape (taps x 128 x
    // 128 channel blocks), not on the kernel's tiling, so a change of tiling leaves the trained weights bit for bit as they were
    const int tiles = nq * cdiv(N, 128) * cdiv(C, 128), kblocks = B * cdiv(out_rows, 32);
    const int splits = max(1, min(64, min(sm_count() / tiles, kblocks / 8)));
    int rc;
    if (N > 64) rc = launch_wgrad<128>(mx, dyt, ld_dyt, dy_sb, B, out_rows, p, splits, st);
    else if (N > 32) rc = launch_wgrad<64>(mx, dyt, ld_dyt, dy_sb, B, out_rows, p, splits, st);
    else rc = launch_wgrad<32>(mx, dyt, ld_dyt, dy_sb, B, out_rows, p, splits, st);
    EVK_REQUIRE(rc != 1, EVK_ERR_UNSUPPORTED, "gconv_wgrad: cuTensorMapEncodeTiled unavailable or rejected the operand");
    if (rc) return rc;
    g_disp_flops[4] += 2.0 * B * (double)out_rows * N * C * nq;
  }
  return EVK_OK;
}

}  // namespace evk

using namespace evk;

extern "C" int evk_set_backend_tma(int32_t on) { g_backend_tma = on ? 1 : 0; return EVK_OK; }
// A/B switches of the TMA kernel (tests / bench): slab = one staged input slab per channel block shared by all taps,
// mt2 = 256-row tiles, trunc_comp = relative accumulator compensation per raw (truncated) operand (0 disables it).
extern "C" int evk_set_tma_options(int32_t slab, int32_t mt2, float trunc_comp) {
  g_opt_slab = slab ? 1 : 0; g_opt_mt2 = mt2 ? 1 : 0; g_trunc_comp = trunc_comp;
  return EVK_OK;
}

extern "C" int evk_gemm_tf32(const float* A, int32_t lda, const float* B, int32_t ldb, float* D, int32_t ldd, int32_t M, int32_t N,
                             int32_t K, const float* bias, const float* res, int32_t ldr, int32_t act, float slope, int32_t splits,
                             cudaStream_t st) {
  EVK_REQUIRE(M > 0 && N > 0 && K > 0, EVK_ERR_ARG, "gemm_tf32: empty problem");
  EVK_REQUIRE((lda % 4) == 0 && (ldb % 4) == 0 && ((((uintptr_t)A) | ((uintptr_t)B)) & 15) == 0, EVK_ERR_ARG,
              "gemm_tf32: operands must be 16-byte aligned with pitches that are multiples of 4 floats");
  EVK_REQUIRE(splits >= 1, EVK_ERR_ARG, "gemm_tf32: splits");
  GemmP p{};
  p.d = D; p.ldd = ldd; p.bias = bias; p.res = res; p.ldr = ldr; p.M = M; p.N = N; p.K = K; p.act = act; p.slope = slope;
  p.atomic = splits > 1 ? 1 : 0;
  p.Z = 1; p.Q = 1; p.P = 1;
  Operands o{A, lda, 0, M, B, ldb, 0, 1, 0, 2};
  p.os = 1; p.o0 = 0;
  int rc = run_gemm(o, p, splits, st);
  EVK_REQUIRE(rc != 1, EVK_ERR_UNSUPPORTED, "gemm_tf32: cuTensorMapEncodeTiled unavailable or rejected the operand");
  if (rc == 0) g_disp_flops[7] += 2.0 * M * (double)N * K;
  return rc;
}

