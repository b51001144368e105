// Stage-1 AR GPT odds and ends: sinusoidal position add (embedding.py:36-81), summed cross-entropy + top-k accuracy
// (t2s_model.py:486-489), and ScaledAdam (optim.py:123-622) over one flat fp32 arena.
#include "evk_common.cuh"

namespace evk {
namespace {

// ------------------------------------------------------------------------------------------------
// y[b][t0 + t][:] = x[b][t][:] + alpha * pe[t][:]
__global__ void sinepos_add_kernel(const float* __restrict__ x, int ldx, long long x_sb, const float* __restrict__ pe, int ldpe,
                                   const float* __restrict__ alpha, float* __restrict__ y, int ldy, long long y_sb, int B,
                                   int T, int D) {
  const float al = alpha[0];
  const int d4 = D / 4;
  const long long n = (long long)B * T * d4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % d4);
    long long r = i / d4;
    int t = (int)(r % T), b = (int)(r / T);
    float4 xv = *reinterpret_cast<const float4*>(x + b * x_sb + (size_t)t * ldx + c * 4);
    float4 pv = *reinterpret_cast<const float4*>(pe + (size_t)t * ldpe + c * 4);
    float4 o = make_float4(xv.x + al * pv.x, xv.y + al * pv.y, xv.z + al * pv.z, xv.w + al * pv.w);
    *reinterpret_cast<float4*>(y + b * y_sb + (size_t)t * ldy + c * 4) = o;
  }
}

// dalpha += sum_{b,t,d} dy[b][t][d] * pe[t][d]
__global__ void sinepos_bwd_kernel(const float* __restrict__ dy, int ldy, long long dy_sb, const float* __restrict__ pe, int ldpe,
                                   float* __restrict__ dalpha, int B, int T, int D) {
  __shared__ float red[33];
  const long long n = (long long)B * T * D;
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int d = (int)(i % D);
    long long r = i / D;
    int t = (int)(r % T), b = (int)(r / T);
    acc += dy[b * dy_sb + (size_t)t * ldy + d] * pe[(size_t)t * ldpe + d];
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) dalpha[blockIdx.x] = acc;            // per-block partial (ordered_sum adds them)
}

// ------------------------------------------------------------------------------------------------
// one warp per row: lse, nll, top-k hit (count of logits strictly above the target logit < k), valid = target != ignore
__global__ void ce_fwd_kernel(const float* __restrict__ logits, int ld, const long long* __restrict__ tgt, int rows, int V,
                              int topk, long long ignore, float* __restrict__ lse, float* __restrict__ nll,
                              unsigned char* __restrict__ flags) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* l = logits + (size_t)row * ld;
  const long long tg = tgt[row];
  float mx = -INFINITY;
  for (int c = lane; c < V; c += 32) mx = fmaxf(mx, l[c]);
  mx = warp_max(mx);
  const float lt = (tg >= 0 && tg < V) ? l[tg] : 0.f;
  float se = 0.f;
  int above = 0;
  for (int c = lane; c < V; c += 32) {
    float v = l[c];
    se += expf(v - mx);
    above += (v > lt) ? 1 : 0;
  }
  se = warp_sum(se);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
  if (lane == 0) {
    float ls = mx + logf(se);
    lse[row] = ls;
    nll[row] = ls - lt;
    const bool valid = tg != ignore;
    flags[row] = (unsigned char)((valid ? 1 : 0) | ((valid && above < topk) ? 2 : 0));
  }
}

// out[0] = sum nll (fixed order), out[1] = hits / max(valid, 1)
__global__ void ce_finalize_kernel(const float* __restrict__ nll, const unsigned char* __restrict__ flags, int rows,
                                   float* __restrict__ out) {
  __shared__ float red[33];
  float s = 0.f, hv = 0.f, vv = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    s += nll[i];
    vv += (flags[i] & 1) ? 1.f : 0.f;
    hv += (flags[i] & 2) ? 1.f : 0.f;
  }
  s = block_sum(s, red);
  hv = block_sum(hv, red);
  vv = block_sum(vv, red);
  if (threadIdx.x == 0) {
    out[0] = s;
    out[1] = hv / fmaxf(vv, 1.f);
  }
}

// dlogits[row][c] = gscale * (exp(l - lse) - [c == tgt])
__global__ void ce_bwd_kernel(const float* __restrict__ logits, int ld, const long long* __restrict__ tgt,
                              const float* __restrict__ lse, const float* __restrict__ gscale, int rows_per_g,
                              float* __restrict__ dl, int lddl, int rows, int V) {
  const long long n = (long long)rows * V;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % V);
    int r = (int)(i / V);
    float p = expf(logits[(size_t)r * ld + c] - lse[r]);
    dl[(size_t)r * lddl + c] = gscale[r / rows_per_g] * (p - ((long long)c == tgt[r] ? 1.f : 0.f));
  }
}

// DPO head (t2s_model.py:421-427, utils.py:160-192, reference_free, beta): A_b = -sum_t nll_c[b][t], R_b = -sum_t nll_r[b][t]
//   loss_2 = mean_b softplus(-beta (A_b - R_b));   out3 = (loss_1 = sum nll_c, loss_2, loss_1 + loss_2)
//   coef_c[b] = d total / d nll_c[b][t] = 1 + beta * sigmoid(-beta (A_b - R_b)) / B ;  coef_r[b] = -(coef_c[b] - 1)
__global__ void dpo_head_kernel(const float* __restrict__ nll_c, int Yc, const float* __restrict__ nll_r, int Yr, int B, float beta,
                                float* __restrict__ out3, float* __restrict__ coef_c, float* __restrict__ coef_r) {
  __shared__ float red[33];
  float l1 = 0.f, l2 = 0.f;
  for (int b = 0; b < B; ++b) {
    float sc = 0.f, sr = 0.f;
    for (int t = threadIdx.x; t < Yc; t += blockDim.x) sc += nll_c[(size_t)b * Yc + t];
    for (int t = threadIdx.x; t < Yr; t += blockDim.x) sr += nll_r[(size_t)b * Yr + t];
    sc = block_sum(sc, red);
    sr = block_sum(sr, red);
    const float z = -beta * ((-sc) - (-sr));                 // -beta (A - R)
    const float sp = z > 0.f ? z + log1pf(expf(-z)) : log1pf(expf(z));
    const float sg = 1.f / (1.f + expf(-z));                 // sigmoid(-beta (A - R))
    l1 += sc; l2 += sp;
    if (threadIdx.x == 0) {
      coef_c[b] = 1.f + beta * sg / (float)B;
      coef_r[b] = -beta * sg / (float)B;
    }
  }
  if (threadIdx.x == 0) {
    out3[0] = l1; out3[1] = l2 / (float)B; out3[2] = l1 + l2 / (float)B;
  }
}

// ------------------------------------------------------------------------------------------------
// ScaledAdam.  chunk table: [nchunks][3] = (tensor id, begin, count) over the flat arenas.
__global__ void sadam_reduce_kernel(const float* __restrict__ p, const float* __restrict__ g, const long long* __restrict__ chunks,
                                    float gscale, float* __restrict__ stats) {
  __shared__ float red[33];
  const long long* ch = chunks + (size_t)blockIdx.x * 3;
  const int t = (int)ch[0];
  const long long beg = ch[1], cnt = ch[2];
  float pp = 0.f, pg = 0.f, gg = 0.f;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    float pv = p[beg + i], gv = g[beg + i] * gscale;
    pp += pv * pv; pg += pv * gv; gg += gv * gv;
  }
  pp = block_sum(pp, red);
  pg = block_sum(pg, red);
  gg = block_sum(gg, red);
  if (threadIdx.x == 0) {                                     // per-chunk partials; sadam_stats_sum adds them in chunk order
    stats[blockIdx.x * 3 + 0] = pp;
    stats[blockIdx.x * 3 + 1] = pg;
    stats[blockIdx.x * 3 + 2] = gg;
  }
}

// stats[t][j] += sum over the chunks c of tensor t (ascending) of part[c][j]
__global__ void sadam_stats_sum_kernel(const float* __restrict__ part, const long long* __restrict__ chunks, int nchunks, int nt,
                                       float* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nt * 3) return;
  const int t = i / 3, j = i - t * 3;
  float acc = 0.f;
  for (int c = 0; c < nchunks; ++c)
    if ((int)chunks[(size_t)c * 3] == t) acc += part[c * 3 + j];
  stats[i] += acc;
}

struct SadamCfg {
  float b1, b2, clip, slr, eps, rmin, rmax;
  int period, sup;
};

__global__ void __launch_bounds__(1024) sadam_scalars_kernel(int nt, const long long* __restrict__ numel, float* __restrict__ stats,
                                                             float* __restrict__ rms, float* __restrict__ sv,
                                                             float* __restrict__ sg, float* __restrict__ coef,
                                                             const float* __restrict__ hyper, long long* __restrict__ stepbuf,
                                                             float* __restrict__ norms, float* __restrict__ thr,
                                                             float* __restrict__ glob, SadamCfg c) {
  __shared__ float red[33];
  __shared__ float srt[1024];
  __shared__ float s_cs;
  const long long step = stepbuf[0];
  const float lr = hyper[0];
  if (step == 0)
    for (int t = threadIdx.x; t < nt; t += blockDim.x)
      if (numel[t] > 1) rms[t] = sqrtf(stats[t * 3] / (float)numel[t]);      // _init_state
  __syncthreads();
  float tot = 0.f;
  for (int t = threadIdx.x; t < nt; t += blockDim.x) tot += (numel[t] > 1 ? rms[t] * rms[t] : 1.f) * stats[t * 3 + 2];
  tot = block_sum(tot, red);
  if (threadIdx.x == 0) s_cs = 1.f;
  __syncthreads();
  if (c.clip > 0.f && step > 0) {
    const float tot_norm = sqrtf(tot);
    if (threadIdx.x == 0) norms[step % c.period] = tot_norm;
    __syncthreads();
    if (step % c.period == 0) {
      srt[threadIdx.x] = (int)threadIdx.x < c.period ? norms[threadIdx.x] : INFINITY;
      __syncthreads();
      for (int k = 2; k <= 1024; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
          int i = threadIdx.x, ixj = i ^ j;
          if (ixj > i) {
            bool up = (i & k) == 0;
            float a = srt[i], b = srt[ixj];
            if ((a > b) == up) { srt[i] = b; srt[ixj] = a; }
          }
          __syncthreads();
        }
      if (threadIdx.x == 0) {
        int idx = min(c.period - 1, (c.period / 4) * 2);
        thr[0] = c.clip * srt[idx];
        thr[1] = 1.f;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0 && step >= c.period && thr[1] != 0.f) s_cs = fminf(1.f, thr[0] / (tot_norm + 1e-20f));
    __syncthreads();
  }
  const float cs = s_cs;
  const int slot = (int)(step % c.sup);
  for (int t = threadIdx.x; t < nt; t += blockDim.x) {
    if (numel[t] > 1) {
      sg[slot * nt + t] = cs * stats[t * 3 + 1];
      float sstep = 0.f;
      if (slot == c.sup - 1) {
        const float r = sqrtf(stats[t * 3] / (float)numel[t]);
        rms[t] = r;
        if (step > 0) {
          const double b2c = pow((double)c.b2, (double)c.sup);
          float msq = 0.f, ssum = 0.f;
          for (int k = 0; k < c.sup; ++k) { float v = sg[k * nt + t]; msq += v * v; ssum += v; }
          msq /= (float)c.sup;
          const float nv = sv[t] * (float)b2c + msq * (float)(1.0 - b2c);
          sv[t] = nv;
          const long long size_step = (step + 1) / c.sup;
          const double bc = 1.0 - pow(b2c, (double)size_step);
          sstep = -(lr * c.slr) * (float)sqrt(bc) * ssum / (sqrtf(nv) + c.eps);
          if (r < c.rmin) sstep = 0.f;
          if (r > c.rmax) sstep = -(lr * c.slr) * (float)c.sup;
        }
      }
      coef[t * 2 + 0] = -lr * (1.f - c.b1) * fmaxf(rms[t], c.rmin);
      coef[t * 2 + 1] = sstep * (1.f - c.b1);
    } else {
      coef[t * 2 + 0] = -(lr * c.slr) * (1.f - c.b1);
      coef[t * 2 + 1] = 0.f;
    }
    stats[t * 3 + 0] = 0.f; stats[t * 3 + 1] = 0.f; stats[t * 3 + 2] = 0.f;
  }
  if (threadIdx.x == 0) {
    const double bc2 = 1.0 - pow((double)c.b2, (double)(step + 1));
    glob[0] = bc2 < 0.99 ? (float)(1.0 / bc2) : 1.f;
    glob[1] = (float)(1.0 / bc2);
    glob[2] = cs;
    stepbuf[0] = step + 1;
  }
}

__global__ void sadam_update_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ delta, float* __restrict__ v,
                                    const long long* __restrict__ chunks, const long long* __restrict__ numel,
                                    const float* __restrict__ coef, const float* __restrict__ glob, float gscale, float b1,
                                    float b2, float eps, float smax, int zero_grad) {
  const long long* ch = chunks + (size_t)blockIdx.x * 3;
  const int t = (int)ch[0];
  const long long beg = ch[1], cnt = ch[2];
  const float alpha = coef[t * 2], sstep = coef[t * 2 + 1];
  const bool scalar = numel[t] == 1;
  const float vs = scalar ? glob[1] : glob[0];
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    const long long e = beg + i;
    const float gv = g[e] * gscale;
    float pv = p[e];
    float d = delta[e] * b1;
    if (!scalar) d += sstep * pv;
    const float vv = v[e] * b2 + (1.f - b2) * gv * gv;
    v[e] = vv;
    d += alpha * gv / (sqrtf(vv * vs) + eps);
    if (scalar) pv = fminf(fmaxf(pv, -smax), smax);
    delta[e] = d;
    p[e] = pv + d;
    if (zero_grad) g[e] = 0.f;
  }
}

// ---- KV-cache attention of one new token (T2SBlock.decode_next_token, t2s_model.py:203-221) --------------------------------
// Cache rows are the in_proj outputs [q | k | v] (3 * H * 32 floats, row pitch ld) of every position so far: rows 0 .. *n_dev, the
// last one just appended; the query is its q block.  The position lives in device memory so that the step can be a replayed CUDA
// graph.  One CTA per (head, batch item), 128 threads, key-parallel (see the kernel).  Exact fp32 -- the sampled token must not
// depend on operand rounding.
// skip (optional, [B][2]): item b never reads keys skip[b][0] .. skip[b][1] - 1 -- the right padding of its text in a batch whose
// rows are padded to a common text length (infer_panel_batch_infer).  The remaining keys are walked as one list, so thread t owns
// the same keys whatever the padding, and a padded key (possibly not finite) never enters a sum.
__global__ void __launch_bounds__(128) attn_decode_kernel(const float* __restrict__ qkv, long long sb, int ld, const int* __restrict__ n_dev,
                                                           const int* __restrict__ skip, int H, float scale, float* __restrict__ out, int ldo) {
  const int n = *n_dev + 1;                                      // keys 0 .. *n_dev
  const int h = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s0 = skip ? skip[2 * b] : n, gap = skip ? skip[2 * b + 1] - s0 : 0;
  const float* base = qkv + (long long)b * sb;
  const int D = H * 32;
  // Key-parallel: thread t owns keys t, t + 128, ... (the whole 32-float q / k / v rows in registers: no per-key shuffle chain,
  // every key's loads are independent -> the ~600-cycle L2 latency is paid once per 128 keys instead of once per key), with a
  // private online softmax; the 128 partial states are merged once at the end.
  float q[32];
  {
    const float4* qp = reinterpret_cast<const float4*>(base + (long long)(n - 1) * ld + h * 32);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float4 t = __ldg(qp + c);
      q[4 * c] = t.x * scale; q[4 * c + 1] = t.y * scale; q[4 * c + 2] = t.z * scale; q[4 * c + 3] = t.w * scale;
    }
  }
  float m = -INFINITY, l = 0.f, acc[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) acc[c] = 0.f;
  for (int t = threadIdx.x; t < n - gap; t += 128) {
    const int j = t < s0 ? t : t + gap;
    const float4* kp = reinterpret_cast<const float4*>(base + (long long)j * ld + D + h * 32);
    const float4* vp = reinterpret_cast<const float4*>(base + (long long)j * ld + 2 * D + h * 32);
    float4 kv[8], vv[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) kv[c] = __ldg(kp + c);
#pragma unroll
    for (int c = 0; c < 8; ++c) vv[c] = __ldg(vp + c);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      s = fmaf(q[4 * c], kv[c].x, fmaf(q[4 * c + 1], kv[c].y, fmaf(q[4 * c + 2], kv[c].z, fmaf(q[4 * c + 3], kv[c].w, s))));
    const float mn = fmaxf(m, s);
    const float c0 = expf(m - mn), p = expf(s - mn);             // m = -inf on the first key: c0 = 0
    l = l * c0 + p;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      acc[4 * c] = fmaf(acc[4 * c], c0, p * vv[c].x); acc[4 * c + 1] = fmaf(acc[4 * c + 1], c0, p * vv[c].y);
      acc[4 * c + 2] = fmaf(acc[4 * c + 2], c0, p * vv[c].z); acc[4 * c + 3] = fmaf(acc[4 * c + 3], c0, p * vv[c].w);
    }
    m = mn;
  }
  // merge: block maximum, rescale, sum l and the 32 output dimensions over the 128 threads
  __shared__ float sm_m[4], sm_r[4][33];
  float M = m;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
  if (lane == 0) sm_m[warp] = M;
  __syncthreads();
  M = fmaxf(fmaxf(sm_m[0], sm_m[1]), fmaxf(sm_m[2], sm_m[3]));
  const float f = (m == -INFINITY) ? 0.f : expf(m - M);          // threads without a key contribute nothing
  l = warp_sum(l * f);
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const float t = warp_sum(acc[c] * f);
    if (lane == c) sm_r[warp][c] = t;
  }
  if (lane == 0) sm_r[warp][32] = l;
  __syncthreads();
  if (warp == 0) {
    const float Ls = sm_r[0][32] + sm_r[1][32] + sm_r[2][32] + sm_r[3][32];
    const float A = sm_r[0][lane] + sm_r[1][lane] + sm_r[2][lane] + sm_r[3][lane];
    out[(long long)b * ldo + h * 32 + lane] = A / Ls;
  }
}

// Skinny product of the AR token step:  y[r][n] = act(sum_c x[r][c] * W[n][c] + bias[n]),  R <= 64 rows.
// A one-row "GEMM" is a stream over the weight matrix (12.6 MB per GPT layer): through the 128-row tensor-core tiles it ran on
// N/128 = 4..16 CTAs with one barrier round trip per 32 channels (25..100 us per Linear, 9.3 ms per token).  Here KS warps share
// one output column (each takes every KS-th float4 group of the weight row: 512-byte coalesced warp loads, four in flight), the x
// rows sit in shared memory, products are exact fp32 FMAs (the sampled token must not depend on operand rounding).
// Rows that do not fit in shared memory at once (R * C floats > the staging budget) are staged CC channels at a time; the weight
// is still read once, and every lane keeps walking its own float4 groups in increasing order across the chunks, so each output's
// FMA chain, its warp sum and the sum over the KS warps are the same for every R: a row's result does not depend on the batch.
template <int R>
__global__ void __launch_bounds__(256) gemv_rows_kernel(const float* __restrict__ x, int ldx, int rows, const float* __restrict__ W, int ldw,
                                                        const float* __restrict__ bias, float* __restrict__ y, int ldy, int N, int C,
                                                        int CC, int KS, int act, float slope) {
  extern __shared__ __align__(16) float gv_x[];                   // [R][CC] staged channels, then [8][R] partial sums
  float* part = gv_x + R * CC;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = 8 / KS;                                          // output columns per CTA
  const int n = blockIdx.x * per + warp / KS, ks = warp % KS;
  const float4* wr = reinterpret_cast<const float4*>(W + (size_t)(n < N ? n : 0) * ldw);
  const int step = 32 * KS;
  int c4 = ks * 32 + lane;                                         // this lane's next float4 group of the weight row
  float acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.f;
  for (int c0 = 0; c0 < C; c0 += CC) {
    const int cc = min(CC, C - c0);
    if (c0) __syncthreads();                                       // every warp is done with the previous chunk
    for (int i = threadIdx.x; i < R * cc; i += blockDim.x) {
      const int r = i / cc, c = i - r * cc;
      gv_x[r * CC + c] = r < rows ? x[(size_t)r * ldx + c0 + c] : 0.f;
    }
    __syncthreads();
    if (n < N) {
      const int g0 = c0 >> 2, g1 = (c0 + cc) >> 2;
      for (; c4 + 3 * step < g1; c4 += 4 * step) {
        float4 w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) w[u] = __ldg(wr + c4 + u * step);
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const float4 xv = reinterpret_cast<const float4*>(gv_x + r * CC)[c4 - g0 + u * step];
            acc[r] = fmaf(w[u].x, xv.x, fmaf(w[u].y, xv.y, fmaf(w[u].z, xv.z, fmaf(w[u].w, xv.w, acc[r]))));
          }
      }
      for (; c4 < g1; c4 += step) {
        const float4 w = __ldg(wr + c4);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 xv = reinterpret_cast<const float4*>(gv_x + r * CC)[c4 - g0];
          acc[r] = fmaf(w.x, xv.x, fmaf(w.y, xv.y, fmaf(w.z, xv.z, fmaf(w.w, xv.w, acc[r]))));
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = warp_sum(acc[r]);
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < R; ++r) part[warp * R + r] = acc[r];
  }
  __syncthreads();
  if (ks == 0 && n < N) {
    for (int r = lane; r < rows && r < R; r += 32) {
      float v = 0.f;
      for (int k = 0; k < KS; ++k) v += part[(warp + k) * R + r];
      if (bias) v += bias[n];
      if (act == EVK_ACT_RELU) v = fmaxf(v, 0.f);
      else if (act == EVK_ACT_LRELU) v = v > 0.f ? v : v * slope;
      y[(size_t)r * ldy + n] = v;
    }
  }
}

// cache[b][*pos][0 .. W) = row[b][0 .. W): the position comes from device memory so that the step can be a replayed CUDA graph
__global__ void cache_append_kernel(const float* __restrict__ row, int ldr, float* __restrict__ cache, long long sb, int ld,
                                    const int* __restrict__ pos, int W) {
  const int b = blockIdx.y;
  float* dst = cache + (long long)b * sb + (long long)(*pos) * ld;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W; i += gridDim.x * blockDim.x) dst[i] = row[(long long)b * ldr + i];
}
}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_sinepos_add(const float* x, int ldx, int64_t x_sb, const float* pe, int ldpe, const float* alpha, float* y,
                               int ldy, int64_t y_sb, int B, int T, int D, cudaStream_t st) {
  EVK_REQUIRE(D % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && ldpe % 4 == 0 && x_sb % 4 == 0 && y_sb % 4 == 0, EVK_ERR_ARG,
              "sinepos_add: D and pitches must be multiples of 4");
  if (B * T == 0) return 0;
  long long n = (long long)B * T * (D / 4);
  sinepos_add_kernel<<<(int)min((long long)kNumSMs * 8, (n + 255) / 256), 256, 0, st>>>(x, ldx, x_sb, pe, ldpe, alpha, y, ldy, y_sb, B, T, D);
  return check_launch("sinepos_add");
}

extern "C" int evk_sinepos_bwd(const float* dy, int ldy, int64_t dy_sb, const float* pe, int ldpe, float* dalpha, int B, int T,
                               int D, cudaStream_t st) {
  if (B * T == 0) return 0;
  long long n = (long long)B * T * D;
  const int blocks = (int)min((long long)kNumSMs * 4, (n + 255) / 256);
  Scratch part_buf(blocks, st);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "sinepos_bwd: scratch allocation failed");
  sinepos_bwd_kernel<<<blocks, 256, 0, st>>>(dy, ldy, dy_sb, pe, ldpe, part, B, T, D);
  if (int rc = check_launch("sinepos_bwd")) return rc;
  return ordered_sum(part, blocks, 1, 1, 1, dalpha, 0, 0, st);
}

extern "C" int evk_ce_fwd(const float* logits, int ld, const int64_t* targets, int rows, int V, int topk, int64_t ignore_index,
                          float* lse, float* nll, uint8_t* flags, float* out2, cudaStream_t st) {
  EVK_REQUIRE(rows > 0 && V > 0, EVK_ERR_ARG, "ce_fwd: empty");
  ce_fwd_kernel<<<cdiv(rows, 8), 256, 0, st>>>(logits, ld, (const long long*)targets, rows, V, topk, ignore_index, lse, nll, flags);
  if (int rc = check_launch("ce_fwd")) return rc;
  ce_finalize_kernel<<<1, 1024, 0, st>>>(nll, flags, rows, out2);
  return check_launch("ce_finalize");
}

extern "C" int evk_dpo_head(const float* nll_c, int Yc, const float* nll_r, int Yr, int B, float beta, float* out3, float* coef_c,
                            float* coef_r, cudaStream_t st) {
  EVK_REQUIRE(B > 0 && Yc > 0 && Yr > 0, EVK_ERR_ARG, "dpo_head: empty");
  dpo_head_kernel<<<1, 256, 0, st>>>(nll_c, Yc, nll_r, Yr, B, beta, out3, coef_c, coef_r);
  return check_launch("dpo_head");
}

extern "C" int evk_ce_bwd(const float* logits, int ld, const int64_t* targets, const float* lse, const float* gscale,
                          int rows_per_g, float* dl, int lddl, int rows, int V, cudaStream_t st) {
  EVK_REQUIRE(rows_per_g > 0, EVK_ERR_ARG, "ce_bwd: rows_per_g");
  long long n = (long long)rows * V;
  ce_bwd_kernel<<<(int)min((long long)kNumSMs * 16, (n + 255) / 256), 256, 0, st>>>(logits, ld, (const long long*)targets, lse, gscale, rows_per_g, dl, lddl, rows, V);
  return check_launch("ce_bwd");
}

extern "C" int evk_scaled_adam(float* p, float* g, float* delta, float* v, const int64_t* chunks, int nchunks,
                               const int64_t* numel, int nt, float* stats, float* rms, float* sv, float* sg, float* coef,
                               const float* hyper, int64_t* stepbuf, float* norms, float* thr, float* glob, float gscale,
                               float beta1, float beta2, float clipping_scale, int clipping_update_period, float scalar_lr_scale,
                               float eps, float param_min_rms, float param_max_rms, float scalar_max, int size_update_period,
                               int zero_grad, cudaStream_t st) {
  EVK_REQUIRE(nt > 0 && nchunks > 0, EVK_ERR_ARG, "scaled_adam: empty");
  EVK_REQUIRE(clipping_update_period >= 1 && clipping_update_period <= 1024, EVK_ERR_UNSUPPORTED,
              "scaled_adam: clipping_update_period %d > 1024", clipping_update_period);
  EVK_REQUIRE(size_update_period >= 1 && size_update_period <= 16, EVK_ERR_UNSUPPORTED, "scaled_adam: size_update_period");
  SadamCfg c{beta1, beta2, clipping_scale, scalar_lr_scale, eps, param_min_rms, param_max_rms, clipping_update_period,
             size_update_period};
  Scratch part_buf(3ll * nchunks, st);
  float* part = part_buf.p;
  EVK_REQUIRE(part, EVK_ERR_CUDA, "scaled_adam: scratch allocation failed");
  sadam_reduce_kernel<<<nchunks, 256, 0, st>>>(p, g, (const long long*)chunks, gscale, part);
  if (int rc = check_launch("sadam_reduce")) return rc;
  sadam_stats_sum_kernel<<<cdiv(3ll * nt, 256), 256, 0, st>>>(part, (const long long*)chunks, nchunks, nt, stats);
  if (int rc = check_launch("sadam_stats_sum")) return rc;
  sadam_scalars_kernel<<<1, 1024, 0, st>>>(nt, (const long long*)numel, stats, rms, sv, sg, coef, hyper, (long long*)stepbuf, norms, thr, glob, c);
  if (int rc = check_launch("sadam_scalars")) return rc;
  sadam_update_kernel<<<nchunks, 256, 0, st>>>(p, g, delta, v, (const long long*)chunks, (const long long*)numel, coef, glob, gscale, beta1, beta2, eps, scalar_max,
                                               zero_grad);
  return check_launch("sadam_update");
}

template <int R>
static int gemv_rows_launch(int grid, size_t smem, cudaStream_t st, const float* x, int ldx, int rows, const float* W, int ldw,
                            const float* bias, float* y, int ldy, int N, int C, int CC, int KS, int act, float slope) {
  if (smem > 48 * 1024) {                                          // opt in once per instance (before any graph capture uses it)
    static unsigned opted = 0;                                     // one bit per device ordinal
    int dev = 0;
    cudaGetDevice(&dev);
    if (!((opted >> (dev & 31)) & 1u)) {
      EVK_REQUIRE(cudaFuncSetAttribute(gemv_rows_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024) == cudaSuccess,
                  EVK_ERR_CUDA, "gemv_rows: shared-memory opt-in failed");
      opted |= 1u << (dev & 31);
    }
  }
  gemv_rows_kernel<R><<<grid, 256, smem, st>>>(x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
  return check_launch("gemv_rows");
}

extern "C" int evk_gemv_rows(const float* x, int32_t ldx, int32_t rows, const float* W, int32_t ldw, const float* bias, float* y,
                             int32_t ldy, int32_t N, int32_t C, int32_t act, float slope, cudaStream_t st) {
  EVK_REQUIRE(x && W && y && rows >= 1 && rows <= 64 && N >= 1 && C >= 4, EVK_ERR_ARG, "gemv_rows: bad arguments (rows=%d N=%d C=%d)", rows, N, C);
  EVK_REQUIRE(C % 4 == 0 && ldw % 4 == 0 && ldw >= C && ((uintptr_t)W % 16) == 0 && ldx >= C && ldy >= N, EVK_ERR_ARG,
              "gemv_rows: C and the weight pitch must be multiples of 4, W 16-byte aligned");
  EVK_REQUIRE(act == EVK_ACT_NONE || act == EVK_ACT_RELU || act == EVK_ACT_LRELU, EVK_ERR_UNSUPPORTED, "gemv_rows: activation %d", act);
  int R = 1;
  while (R < rows) R *= 2;
  // <= 4 rows: all C channels staged at once (40 KB at most); more rows: chunks of CC channels in a 64 KB staging buffer
  int CC = C;
  if (R <= 4) EVK_REQUIRE((size_t)R * C * 4 <= 40 * 1024, EVK_ERR_UNSUPPORTED, "gemv_rows: %d rows of %d channels exceed the staging buffer", R, C);
  else CC = min(C, (64 * 1024 / 4 / R) & ~3);
  int KS = 1;
  while (KS < 8 && (long long)N * KS < kNumSMs * 8 && C / 4 >= 64 * KS) KS *= 2;      // enough warps to cover the chip, >= 2 float4 groups per lane
  const int per = 8 / KS;
  const size_t smem = ((size_t)R * CC + 8 * R) * sizeof(float);
  const int grid = cdiv(N, per);
  switch (R) {
    case 1: return gemv_rows_launch<1>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    case 2: return gemv_rows_launch<2>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    case 4: return gemv_rows_launch<4>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    case 8: return gemv_rows_launch<8>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    case 16: return gemv_rows_launch<16>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    case 32: return gemv_rows_launch<32>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
    default: return gemv_rows_launch<64>(grid, smem, st, x, ldx, rows, W, ldw, bias, y, ldy, N, C, CC, KS, act, slope);
  }
}

extern "C" int evk_attn_decode_dev(const float* qkv, int64_t batch_stride, int32_t ld, const int32_t* n_prev_dev, const int32_t* skip,
                                   int32_t B, int32_t H, float scale, float* out, int32_t ldo, cudaStream_t st) {
  EVK_REQUIRE(qkv && out && n_prev_dev && B >= 1 && H >= 1, EVK_ERR_ARG, "attn_decode_dev: bad arguments");
  EVK_REQUIRE(ld >= 3 * H * 32 && ldo >= H * 32, EVK_ERR_ARG, "attn_decode_dev: row pitch %d / %d too small for %d heads of 32", ld, ldo, H);
  EVK_REQUIRE(ld % 4 == 0 && batch_stride % 4 == 0 && ((uintptr_t)qkv % 16) == 0, EVK_ERR_ARG, "attn_decode_dev: rows must be 16-byte aligned");
  attn_decode_kernel<<<dim3(H, B), 128, 0, st>>>(qkv, batch_stride, ld, n_prev_dev, skip, H, scale, out, ldo);
  return check_launch("attn_decode_dev");
}

extern "C" int evk_cache_append(const float* row, int32_t ldr, float* cache, int64_t batch_stride, int32_t ld, const int32_t* pos_dev,
                                int32_t B, int32_t W, cudaStream_t st) {
  EVK_REQUIRE(row && cache && pos_dev && B >= 1 && W >= 1 && W <= ld && W <= ldr, EVK_ERR_ARG, "cache_append: bad arguments");
  cache_append_kernel<<<dim3(cdiv(W, 256), B), 256, 0, st>>>(row, ldr, cache, batch_stride, ld, pos_dev, W);
  return check_launch("cache_append");
}
