// Fused token sampler of the stage-1 GPT's KV-cache decoding (Text2SemanticDecoder.infer_panel_batch_infer, t2s_model.py:563-730,
// and infer_panel_naive, :762-867, which also runs the prompt-free rows of infer_panel_naive_batched):
// one CTA per batch row does the whole of utils.py:109-157 on that row's logits, appends the token to the row's history and
// writes the next input row, so a decode step needs no host round trip and replays as part of one CUDA graph.
// evk_sample_tokens reads one configuration for the whole batch; evk_sample_tokens_rows (tts.run_many, which decodes rows of
// several requests together) reads one per row, including the row's own noise key.
#include <float.h>
#include <limits.h>

#include "evk_common.cuh"

namespace evk {
namespace {

constexpr int kSampThreads = 1024;
constexpr int kSampMaxV = 2048;
constexpr int kSampRowI = 8, kSampRowF = 4;        // row pitches of evk_sample_tokens_rows' tables

__device__ __forceinline__ bool better(float v2, int i2, float v, int i) { return v2 > v || (v2 == v && i2 < i); }

// block-wide (max value, lowest index among equal values); the order (value desc, index asc) is total, so the result does not
// depend on the reduction tree.  rv / ri: >= 33 entries.
__device__ __forceinline__ void block_argmax(float& v, int& i, float* rv, int* ri) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(v2, i2, v, i)) { v = v2; i = i2; }
  }
  __syncthreads();
  if (lane == 0) { rv[w] = v; ri[w] = i; }
  __syncthreads();
  if (w == 0) {
    v = lane < nw ? rv[lane] : -INFINITY;
    i = lane < nw ? ri[lane] : INT_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
      if (better(v2, i2, v, i)) { v = v2; i = i2; }
    }
    if (lane == 0) { rv[32] = v; ri[32] = i; }
  }
  __syncthreads();
  v = rv[32];
  i = ri[32];
}

__global__ void __launch_bounds__(kSampThreads) sample_tokens_kernel(
    const float* __restrict__ logits, int ldl, int V, int eos, int eos_steps, const long long* __restrict__ icfg, int ics,
    const float* __restrict__ fcfg, int fcs, const int* __restrict__ n_dev, const float* __restrict__ q, int ldq, long long* __restrict__ hist, int ldh,
    unsigned* __restrict__ seen, int* __restrict__ fin, const float* __restrict__ emb, const float* __restrict__ pe,
    const float* __restrict__ alpha, float* __restrict__ x_next, int D) {
  __shared__ float pl[kSampMaxV];        // penalised logits (the EOS test's argmax sees them, like the reference's in-place scatter_)
  __shared__ float pr[kSampMaxV];        // softmax of pl (top-p)
  __shared__ float fl[kSampMaxV];        // after top-p and temperature
  __shared__ float red[33];
  __shared__ float rv[33];
  __shared__ int ri[33];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (fin[2 * b] >= 0) return;                                   // a finished row is frozen
  // ics / fcs: 0 when every row reads the one configuration, else the row pitch of the per-row table, whose entries 6 and 7
  // are the row's EOS-exclusion steps and the row index its noise is keyed by
  icfg += (size_t)b * ics;
  fcfg += (size_t)b * fcs;
  const int prefix = (int)icfg[1], n0 = (int)icfg[2], top_k = (int)icfg[3], early = (int)icfg[4], max_steps = (int)icfg[5];
  const int eos_st = ics ? (int)icfg[6] : eos_steps, key_row = ics ? (int)icfg[7] : b;
  const float top_p = fcfg[0], temp = fmaxf(fcfg[1], 1e-5f), pen = fcfg[2];
  const int idx = *n_dev - n0;                                   // decoding step of this replay
  const int W = (V + 31) >> 5;
  const unsigned* sb = seen + (size_t)b * W;
  // 1. repetition penalty over the row's history, prompt included (utils.py:117-123); steps idx < eos_st leave EOS out
  //    (infer_panel_batch_infer: step 0 only, :651-652; infer_panel_naive: the first 11 steps, :835-836)
  for (int i = tid; i < V; i += blockDim.x) {
    float l = logits[(size_t)b * ldl + i];
    if ((sb[i >> 5] >> (i & 31)) & 1u) l = l < 0.f ? l * pen : l / pen;
    pl[i] = (idx < eos_st && i == eos) ? -INFINITY : l;
  }
  __syncthreads();
  float amv = -INFINITY;
  int ami = INT_MAX;
  for (int i = tid; i < V; i += blockDim.x)
    if (better(pl[i], i, amv, ami)) { amv = pl[i]; ami = i; }
  block_argmax(amv, ami, rv, ri);                                // argmax of the penalised logits (:668)
  // 2. nucleus cut (utils.py:125-135) on the penalised, un-tempered logits: in descending order (ties by index), drop every
  //    element whose cumulative probability exceeds top_p, the first one excepted.  cum_i = sum of p_j over the j sorted at or
  //    before i, summed in index order.
  if (top_p < 1.f) {
    float z = 0.f;
    for (int i = tid; i < V; i += blockDim.x) z += expf(pl[i] - amv);
    z = block_sum(z, red);
    for (int i = tid; i < V; i += blockDim.x) pr[i] = expf(pl[i] - amv) / z;
    __syncthreads();
    for (int i = tid; i < V; i += blockDim.x) {
      const float li = pl[i];
      float cum = 0.f;
      for (int j = 0; j < V; ++j) {
        const float lj = pl[j];
        if (lj > li || (lj == li && j <= i)) cum += pr[j];
      }
      fl[i] = (cum > top_p && i != ami) ? -INFINITY : li / temp;
    }
  } else {
    for (int i = tid; i < V; i += blockDim.x) fl[i] = pl[i] / temp;
  }
  __syncthreads();
  // 3. top-k (utils.py:139-142): keep every value >= the k-th largest, ties included  <=>  fewer than k values strictly above it
  const int k = min(top_k, V);
  float mx = -INFINITY;
  int mi = INT_MAX;
  for (int i = tid; i < V; i += blockDim.x) {
    const float fi = fl[i];
    int c = 0;
    for (int j = 0; j < V && c < k; ++j) c += fl[j] > fi;
    const float f = c < k ? fi : -INFINITY;
    pl[i] = f;                                                   // pl is free again: it now holds the top-k filtered logits
    if (better(f, i, mx, mi)) { mx = f; mi = i; }
  }
  block_argmax(mx, mi, rv, ri);
  // 4. softmax, then argmax(p / q) with q ~ Exp(1) (utils.py:102-106).  q: supplied [B][ldq], or a counter-based draw keyed by
  //    (seed, key row, step, vocabulary id)
  float s = 0.f;
  for (int i = tid; i < V; i += blockDim.x) s += expf(pl[i] - mx);
  s = block_sum(s, red);
  const Philox ph((uint64_t)icfg[0]);
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int i = tid; i < V; i += blockDim.x) {
    float qi;
    if (q) {
      qi = q[(size_t)b * ldq + i];
    } else {
      const uint4 r = ph(((uint64_t)(unsigned)idx << 32) | (unsigned)i, (uint64_t)key_row);
      qi = -logf(((r.x >> 8) + 0.5f) * (1.0f / 16777216.0f));    // u in (0, 1): q in (0, 17)
    }
    const float sc = (expf(pl[i] - mx) / s) / qi;
    if (better(sc, i, bv, bi)) { bv = sc; bi = i; }
  }
  block_argmax(bv, bi, rv, ri);
  const int tok = bi;
  // 5. append, EOS test, early stop / step cap (t2s_model.py:662-700)
  const bool stop_eos = tok == eos || ami == eos;
  const bool stop_len = (early != -1 && idx + 1 > early) || idx == max_steps - 1;
  if (tid == 0) {
    hist[(size_t)b * ldh + prefix + idx] = tok;
    seen[(size_t)b * W + (tok >> 5)] |= 1u << (tok & 31);
    if (stop_eos) { fin[2 * b] = idx; fin[2 * b + 1] = idx - 1; }
    else if (stop_len) { fin[2 * b] = idx; fin[2 * b + 1] = idx; }
  }
  if (stop_eos || stop_len) return;
  // 6. next input row: emb[token] * x_scale (= 1) + alpha * pe[prefix + idx] (t2s_model.py:705), rounded as torch does
  const float a = alpha[0];
  const float* er = emb + (size_t)tok * D;
  const float* pr_ = pe + (size_t)(prefix + idx) * D;
  for (int c = tid; c < D; c += blockDim.x) x_next[(size_t)b * D + c] = __fadd_rn(er[c], __fmul_rn(a, pr_[c]));
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_sample_tokens(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, int32_t eos_steps,
                                 const int64_t* icfg, const float* fcfg, const int32_t* n_dev, const float* q, int32_t ldq,
                                 int64_t* hist, int32_t ldh, uint32_t* seen, int32_t* fin, const float* emb, const float* pe,
                                 const float* alpha, float* x_next, int32_t D, cudaStream_t st) {
  EVK_REQUIRE(logits && icfg && fcfg && n_dev && hist && seen && fin && emb && pe && alpha && x_next, EVK_ERR_ARG,
              "sample_tokens: null argument");
  EVK_REQUIRE(B >= 1 && V >= 2 && V <= kSampMaxV && eos >= 0 && eos < V && ldl >= V && D >= 1 && (!q || ldq >= V), EVK_ERR_ARG,
              "sample_tokens: bad shape (B=%d V=%d eos=%d ldl=%d)", B, V, eos, ldl);
  EVK_REQUIRE(eos_steps >= 0, EVK_ERR_ARG, "sample_tokens: eos_steps must be >= 0, got %d", eos_steps);
  sample_tokens_kernel<<<B, kSampThreads, 0, st>>>(logits, ldl, V, eos, eos_steps, (const long long*)icfg, 0, fcfg, 0, n_dev, q,
                                                   ldq, (long long*)hist, ldh, seen, fin, emb, pe, alpha, x_next, D);
  return check_launch("sample_tokens");
}

extern "C" int evk_sample_tokens_rows(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, const int64_t* icfg,
                                      const float* fcfg, const int32_t* n_dev, int64_t* hist, int32_t ldh, uint32_t* seen,
                                      int32_t* fin, const float* emb, const float* pe, const float* alpha, float* x_next, int32_t D,
                                      cudaStream_t st) {
  EVK_REQUIRE(logits && icfg && fcfg && n_dev && hist && seen && fin && emb && pe && alpha && x_next, EVK_ERR_ARG,
              "sample_tokens_rows: null argument");
  EVK_REQUIRE(B >= 1 && V >= 2 && V <= kSampMaxV && eos >= 0 && eos < V && ldl >= V && D >= 1, EVK_ERR_ARG,
              "sample_tokens_rows: bad shape (B=%d V=%d eos=%d ldl=%d)", B, V, eos, ldl);
  sample_tokens_kernel<<<B, kSampThreads, 0, st>>>(logits, ldl, V, eos, 0, (const long long*)icfg, kSampRowI, fcfg, kSampRowF,
                                                   n_dev, nullptr, 0, (long long*)hist, ldh, seen, fin, emb, pe, alpha, x_next, D);
  return check_launch("sample_tokens_rows");
}
