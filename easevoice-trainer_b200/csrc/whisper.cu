// Whisper transcription (whisper.py, asr.py), inference only.  The encoder and the decoder's Linears, LayerNorms and the
// encoder's attention run on the library's existing kernels; this file holds what they lack:
//   logmel_kernel / logmel_max_kernel / logmel_norm_kernel
//                                       the 400-point periodic-Hann STFT (hop 160, centre reflect padding) as a direct DFT
//                                       against a precomputed basis, |X|^2, the Slaney mel bank, log10(max(., 1e-10)) over
//                                       whole clips of any length; partial maxima per 256 frames, combined in a fixed order
//                                       per clip; then max(x, clip max - 8), (x + 4) / 4 over each clip's own frames, zero
//                                       after them
//   embed_kernel / add_pos_kernel       token + learned position rows; the encoder's sinusoidal positions
//   self_kv_kernel                      a row's new self-attention K / V written once into its slot, listed in its slot table
//   attn_kernel                         head-dim-64 decode attention in exact fp32: one query row against its slot table, or
//                                       the beams of a clip against the clip's cross-attention keys (read once per block)
//   row_layernorm_kernel                LayerNorm of any width, one row per block (large-v3 has 1280 channels)
//   first_pass_kernel                   no-speech probability and the language argmax at <|startoftranscript|>
//   cand_kernel / merge_kernel          the beam step: transformers' logits processors on the log-softmax, per-row top
//                                       candidates, then the per-clip merge of GenerationMixin._beam_search; optionally the
//                                       log-sum-exp of each processed row summed along every hypothesis (long-form
//                                       avg_logprob)
//   window_kernel                       30 s windows [seek, seek + n) of whole-clip log-mels, zero after n
#include <math.h>

#include "evk_common.cuh"

namespace evk {
namespace {

constexpr int kNfft = 400, kHop = 160, kBins = 201, kFrames = 3000;
constexpr int kFpb = 16;                       // frames per logmel block
constexpr int kMaxBeam = 8, kMaxLd = 448, kMaxK = 16;

// One block per (16 frames t0 .. t0 + 15, clip) of a [B][T][M] buffer, the whole clip, any length: thread k < 201 owns DFT bin
// k for all 16 frames; the basis is [400][201] (cos | sin, window folded in), so a warp reads consecutive bins.  Frame t of
// clip b (n samples, nf frames) goes to out + (b T + t) M; frames past nf are not written.
__global__ void __launch_bounds__(256) logmel_kernel(const float* __restrict__ wav, long long ldw, const int* __restrict__ lens,
                                                     const float* __restrict__ cosb, const float* __restrict__ sinb,
                                                     const float* __restrict__ fb, int M, int T, float* __restrict__ out) {
  const int b = blockIdx.y, t0 = blockIdx.x * kFpb, n = lens[b], nf = n / kHop;
  if (t0 >= nf) return;
  const float* x = wav + (long long)b * ldw;
  out += (long long)b * T * M;
  __shared__ float fr[kFpb][kNfft];
  __shared__ float pw[kFpb][kBins + 1];
  for (int e = threadIdx.x; e < kFpb * kNfft; e += blockDim.x) {
    const int f = e / kNfft, i = e - f * kNfft;
    long long s = (long long)(t0 + f) * kHop + i - kNfft / 2;   // reflect about the first and last sample
    if (s < 0) s = -s;
    if (s >= n) s = 2 * (long long)(n - 1) - s;
    s = s < 0 ? 0 : (s >= n ? n - 1 : s);                   // clips shorter than 201 samples are rejected by the caller
    fr[f][i] = (t0 + f < nf) ? x[s] : 0.f;
  }
  __syncthreads();
  const int k = threadIdx.x;
  if (k < kBins) {
    float re[kFpb], im[kFpb];
#pragma unroll
    for (int f = 0; f < kFpb; ++f) re[f] = im[f] = 0.f;
    for (int i = 0; i < kNfft; ++i) {
      const float c = cosb[i * kBins + k], s = sinb[i * kBins + k];
#pragma unroll
      for (int f = 0; f < kFpb; ++f) {
        re[f] = fmaf(fr[f][i], c, re[f]);
        im[f] = fmaf(fr[f][i], s, im[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < kFpb; ++f) pw[f][k] = re[f] * re[f] + im[f] * im[f];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kFpb * M; e += blockDim.x) {
    const int f = e / M, m = e - f * M;
    if (t0 + f >= nf) continue;
    float acc = 0.f;
    for (int q = 0; q < kBins; ++q) acc = fmaf(pw[f][q], fb[q * M + m], acc);
    out[(long long)(t0 + f) * M + m] = log10f(fmaxf(acc, 1e-10f));
  }
}

constexpr int kMaxChunk = 256;                 // frames per partial maximum

// One block per (256 frames, clip): part[b][c] = the max over the clip's frames [256 c, 256 c + 256) (-inf past its end).
__global__ void __launch_bounds__(256) logmel_max_kernel(const int* __restrict__ lens, int M, int T, const float* __restrict__ lm,
                                                         float* __restrict__ part) {
  __shared__ float red[33];
  const int b = blockIdx.y, c = blockIdx.x, nf = lens[b] / kHop;
  const int f0 = c * kMaxChunk, f1 = min(nf, f0 + kMaxChunk);
  const float* o = lm + (long long)b * T * M;
  float mx = -INFINITY;
  for (long long e = (long long)f0 * M + threadIdx.x; e < (long long)f1 * M; e += blockDim.x) mx = fmaxf(mx, o[e]);
  mx = block_max(mx, red);
  if (threadIdx.x == 0) part[(long long)b * gridDim.x + c] = mx;
}

// Blocks (slice, clip): every block folds its clip's partial maxima in chunk order, then clamps and scales its slice of
// frames; frames from the clip's num_frames to T are zeroed.
__global__ void __launch_bounds__(256) logmel_norm_kernel(const int* __restrict__ lens, int M, int T, int n_part,
                                                          const float* __restrict__ part, float* __restrict__ lm) {
  const int b = blockIdx.y, nf = lens[b] / kHop;
  float mx = -INFINITY;
  for (int c = 0; c < n_part; ++c) mx = fmaxf(mx, part[(long long)b * n_part + c]);
  const float lo = mx - 8.f;
  float* o = lm + (long long)b * T * M;
  const long long nv = (long long)nf * M, nall = (long long)T * M;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < nall; e += (long long)gridDim.x * blockDim.x)
    o[e] = e < nv ? (fmaxf(o[e], lo) + 4.f) * 0.25f : 0.f;
}

// Blocks (frame group, output row): row r is frames [seek, seek + n) of clip row tab[r] = (clip, seek, n), zero after n
// (and past the source's T frames).
__global__ void __launch_bounds__(256) window_kernel(const float* __restrict__ lm, int T, int M, const int* __restrict__ tab,
                                                     float* __restrict__ out) {
  const int r = blockIdx.y, clip = tab[3 * r], seek = tab[3 * r + 1], n = tab[3 * r + 2];
  const float* src = lm + ((long long)clip * T + seek) * M;
  float* dst = out + (long long)r * kFrames * M;
  const long long e1 = (long long)min(kFrames, (blockIdx.x + 1) * kFpb) * M;
  const long long nv = (long long)min(n, T - seek) * M;
  for (long long e = (long long)blockIdx.x * kFpb * M + threadIdx.x; e < e1; e += blockDim.x) dst[e] = e < nv ? src[e] : 0.f;
}

__global__ void embed_kernel(const int* __restrict__ tok, const float* __restrict__ emb, const float* __restrict__ pe,
                             const int* __restrict__ pos, int d, float* __restrict__ x) {
  const int r = blockIdx.x, p = *pos;
  const float* e = emb + (long long)tok[r] * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) x[(long long)r * d + c] = e[c] + pe[(long long)p * d + c];
}

__global__ void add_pos_kernel(float* __restrict__ x, long long rows, int T, int d, const float* __restrict__ pe) {
  const long long n = rows * d;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / d;
    x[e] += pe[(r % T) * d + (e - r * d)];
  }
}

// row r: k | v (columns [d, 3d) of its QKV row) into slot r * S + pos of the layer's pool block; tab[r][pos] = that slot
__global__ void self_kv_kernel(const float* __restrict__ qkv, int ldq, int d, float* __restrict__ pool, long long ldp,
                               int* __restrict__ tab, int ld_tab, const int* __restrict__ pos, int S) {
  const int r = blockIdx.x, p = *pos, slot = r * S + p;
  for (int c = threadIdx.x; c < 2 * d; c += blockDim.x) pool[(long long)slot * ldp + c] = qkv[(long long)r * ldq + d + c];
  if (threadIdx.x == 0) tab[(long long)r * ld_tab + p] = slot;
}

// Block (group, head): nq query rows q0 .. q0 + nq - 1 that share their keys.  Slot-table mode (tab != null, nq == 1): keys
// j <= *pos at rows tab[q0][j].  Cross mode: keys j < n_keys at rows group * n_keys + j.  Scores in shared memory, softmax in
// fp32 with expf, then each output column summed over the keys in two interleaved halves added in a fixed order: the result
// of a row depends on nothing but its own query and keys.
__global__ void __launch_bounds__(128) attn_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ kv,
                                                   long long ldkv, int v_off, const int* __restrict__ tab, int ld_tab,
                                                   const int* __restrict__ pos, int n_keys, int nq, float scale,
                                                   float* __restrict__ o, int ldo) {
  extern __shared__ float sm[];
  const int g = blockIdx.x, h = blockIdx.y, tid = threadIdx.x;
  const int L = tab ? *pos + 1 : n_keys, q0 = g * nq;
  float* sq = sm;                                // [nq][64]
  float* sc = sm + nq * 64;                      // [nq][L]
  __shared__ float red[2][64 * kMaxBeam];
  __shared__ float stat[kMaxBeam][2];
  for (int e = tid; e < nq * 64; e += 128) sq[e] = q[(long long)(q0 + e / 64) * ldq + h * 64 + (e & 63)] * scale;
  __syncthreads();
  auto krow = [&](int j) -> long long { return tab ? (long long)tab[(long long)q0 * ld_tab + j] : (long long)g * n_keys + j; };
  for (int j = tid; j < L; j += 128) {
    const float4* k4 = reinterpret_cast<const float4*>(kv + krow(j) * ldkv + h * 64);
    float kr[64];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float4 v = k4[i];
      kr[4 * i] = v.x; kr[4 * i + 1] = v.y; kr[4 * i + 2] = v.z; kr[4 * i + 3] = v.w;
    }
    for (int a = 0; a < nq; ++a) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 64; ++i) s = fmaf(sq[a * 64 + i], kr[i], s);
      sc[a * L + j] = s;
    }
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int a = warp; a < nq; a += 4) {            // one warp per query row: max, then exp and sum
    float m = -INFINITY;
    for (int j = lane; j < L; j += 32) m = fmaxf(m, sc[a * L + j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float e = expf(sc[a * L + j] - m);
      sc[a * L + j] = e;
      s += e;
    }
    s = warp_sum(s);
    if (lane == 0) stat[a][0] = s;
  }
  __syncthreads();
  const int c = tid & 63, half = tid >> 6;
  float acc[kMaxBeam];
#pragma unroll
  for (int a = 0; a < kMaxBeam; ++a) acc[a] = 0.f;
  for (int j = half; j < L; j += 2) {
    const float v = kv[krow(j) * ldkv + v_off + h * 64 + c];
#pragma unroll
    for (int a = 0; a < kMaxBeam; ++a)
      if (a < nq) acc[a] = fmaf(sc[a * L + j], v, acc[a]);
  }
#pragma unroll
  for (int a = 0; a < kMaxBeam; ++a)
    if (a < nq) red[half][a * 64 + c] = acc[a];
  __syncthreads();
  if (half == 0)
    for (int a = 0; a < nq; ++a) o[(long long)(q0 + a) * ldo + h * 64 + c] = (red[0][a * 64 + c] + red[1][a * 64 + c]) / stat[a][0];
}

// LayerNorm of one row per block, any width (large-v3's 1280 channels exceed evk_layernorm_fwd's 1024): mean, then the
// centred variance, each summed thread-strided and reduced in a fixed order, so a row's bits do not depend on the batch.
__global__ void __launch_bounds__(256) row_layernorm_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, float* __restrict__ y,
                                                            int ldy, int C) {
  __shared__ float red[33];
  const float* xr = x + (long long)blockIdx.x * ldx;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s += xr[c];
  const float mean = block_sum(s, red) / (float)C;
  float q = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = xr[c] - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q, red) / (float)C + eps);
  float* yr = y + (long long)blockIdx.x * ldy;
  for (int c = threadIdx.x; c < C; c += blockDim.x) yr[c] = (xr[c] - mean) * rstd * gamma[c] + beta[c];
}

// one block per row: softmax probability of the no-speech token, argmax over the language tokens (the lowest id on a tie)
__global__ void __launch_bounds__(512) first_pass_kernel(const float* __restrict__ lg, long long ld, int V, int nospeech,
                                                         const int* __restrict__ lang_ids, int n_lang, float* __restrict__ nsp,
                                                         int* __restrict__ lang_tok) {
  __shared__ float red[33];
  const float* x = lg + (long long)blockIdx.x * ld;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, x[v]);
  m = block_max(m, red);
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(x[v] - m);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    nsp[blockIdx.x] = expf(x[nospeech] - m) / s;
    int best = lang_ids[0];
    for (int i = 1; i < n_lang; ++i) {
      const int t = lang_ids[i];
      if (x[t] > x[best] || (x[t] == x[best] && t < best)) best = t;
    }
    lang_tok[blockIdx.x] = best;
  }
}

struct Cand { float v; int i; };
__device__ __forceinline__ bool better(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

struct StepCfg {
  int V, eot, notimestamps, ts_begin, max_init_ts;       // max_init_ts < 0: none
  const int* sup; int n_sup; const int* bsup; int n_bsup;
};

// The processed log-probability of token v for a row (transformers: log_softmax, then SuppressTokensAtBegin, SuppressTokens,
// WhisperTimeStamp).  lp = x - m - log(s); rules: see whisper_oracle.process.
struct RowRules { int first, mask_ts, mask_text_below_eot, ts_lim, force_ts; };

__device__ __forceinline__ bool suppressed(const unsigned* bits, int v) { return (bits[v >> 5] >> (v & 31)) & 1u; }

__device__ __forceinline__ float masked_lp(float lp, int v, const RowRules& R, const StepCfg& c, const unsigned* bits) {
  if (suppressed(bits, v) || v == c.notimestamps) return -INFINITY;
  if (R.mask_ts && v >= c.ts_begin) return -INFINITY;
  if (R.mask_text_below_eot && v < c.eot) return -INFINITY;
  if (v >= c.ts_begin && v < R.ts_lim) return -INFINITY;
  if (R.first) {
    if (v < c.ts_begin) return -INFINITY;
    if (c.max_init_ts >= 0 && v > c.ts_begin + c.max_init_ts) return -INFINITY;
  }
  if (R.force_ts && v < c.ts_begin) return -INFINITY;
  return lp;
}

// One block per row (512 threads): the row's processed log-probs plus its running score, top K (value, token) candidates,
// best first, the lower token first on a tie.
__global__ void __launch_bounds__(512) cand_kernel(const float* __restrict__ lg, long long ld, StepCfg c,
                                                   const int* __restrict__ hist, int ld_hist, const int* __restrict__ gstep,
                                                   const float* __restrict__ run_score, int K, float* __restrict__ cv,
                                                   int* __restrict__ ci, float* __restrict__ row_lse) {
  extern __shared__ unsigned bits[];             // [ceil(V / 32)]
  __shared__ float red[33];
  __shared__ RowRules R;
  __shared__ Cand heads[512];
  const int r = blockIdx.x, tid = threadIdx.x, g = *gstep, nw = (c.V + 31) >> 5;
  const float* x = lg + (long long)r * ld;
  for (int i = tid; i < nw; i += blockDim.x) bits[i] = 0u;
  __syncthreads();
  for (int i = tid; i < c.n_sup; i += blockDim.x) if (c.sup[i] < c.V) atomicOr(&bits[c.sup[i] >> 5], 1u << (c.sup[i] & 31));
  if (g == 0)
    for (int i = tid; i < c.n_bsup; i += blockDim.x) if (c.bsup[i] < c.V) atomicOr(&bits[c.bsup[i] >> 5], 1u << (c.bsup[i] & 31));
  if (tid == 0) {
    const int* hr = hist + (long long)r * ld_hist;
    const bool last_ts = g >= 1 && hr[g - 1] >= c.ts_begin;
    const bool pen_ts = g < 2 || hr[g - 2] >= c.ts_begin;
    R.first = g == 0;
    R.mask_ts = last_ts && pen_ts;
    R.mask_text_below_eot = last_ts && !pen_ts;
    int lt = -1;
    for (int i = g - 1; i >= 0; --i) if (hr[i] >= c.ts_begin) { lt = hr[i]; break; }
    R.ts_lim = lt < 0 ? c.ts_begin : ((last_ts && !pen_ts) ? lt : lt + 1);
    R.force_ts = 0;
  }
  __syncthreads();
  // log_softmax of the raw logits
  float m = -INFINITY;
  for (int v = tid; v < c.V; v += blockDim.x) m = fmaxf(m, x[v]);
  m = block_max(m, red);
  float s = 0.f;
  for (int v = tid; v < c.V; v += blockDim.x) s += expf(x[v] - m);
  const float ls = logf(block_sum(s, red));
  RowRules Rl = R;
  // the timestamp processor's own log_softmax of the masked scores, then logsumexp over timestamps vs the best text token
  float m2 = -INFINITY;
  for (int v = tid; v < c.V; v += blockDim.x) m2 = fmaxf(m2, masked_lp((x[v] - m) - ls, v, Rl, c, bits));
  m2 = block_max(m2, red);
  float s2 = 0.f;
  for (int v = tid; v < c.V; v += blockDim.x) {
    const float a = masked_lp((x[v] - m) - ls, v, Rl, c, bits);
    s2 += a == -INFINITY ? 0.f : expf(a - m2);
  }
  const float ls2 = logf(block_sum(s2, red));
  float mt = -INFINITY, mx = -INFINITY;
  for (int v = tid; v < c.V; v += blockDim.x) {
    const float l2 = (masked_lp((x[v] - m) - ls, v, Rl, c, bits) - m2) - ls2;
    if (v >= c.ts_begin) mt = fmaxf(mt, l2); else mx = fmaxf(mx, l2);
  }
  mt = block_max(mt, red);
  mx = block_max(mx, red);
  float st = 0.f;
  if (mt != -INFINITY)
    for (int v = c.ts_begin + tid; v < c.V; v += blockDim.x) {
      const float l2 = (masked_lp((x[v] - m) - ls, v, Rl, c, bits) - m2) - ls2;
      st += l2 == -INFINITY ? 0.f : expf(l2 - mt);
    }
  st = block_sum(st, red);
  const float ts_lse = mt == -INFINITY ? -INFINITY : mt + logf(st);
  Rl.force_ts = ts_lse > mx;
  if (row_lse) {                                 // log-sum-exp of the processed row: its log_softmax is lp - this
    float m3 = -INFINITY;
    for (int v = tid; v < c.V; v += blockDim.x) m3 = fmaxf(m3, masked_lp((x[v] - m) - ls, v, Rl, c, bits));
    m3 = block_max(m3, red);
    float s3 = 0.f;
    for (int v = tid; v < c.V; v += blockDim.x) {
      const float a = masked_lp((x[v] - m) - ls, v, Rl, c, bits);
      s3 += a == -INFINITY ? 0.f : expf(a - m3);
    }
    s3 = block_sum(s3, red);
    if (tid == 0) row_lse[r] = m3 + logf(s3);
  }
  // candidates: per-thread sorted top K, then K rounds of a block argmax over the threads' heads
  const float base = run_score[r];
  Cand top[kMaxK];
  for (int k = 0; k < K; ++k) top[k] = Cand{-INFINITY, 0x7fffffff};
  for (int v = tid; v < c.V; v += blockDim.x) {
    const float a = masked_lp((x[v] - m) - ls, v, Rl, c, bits) + base;
    if (!better(a, v, top[K - 1].v, top[K - 1].i)) continue;
    int k = K - 1;
    while (k > 0 && better(a, v, top[k - 1].v, top[k - 1].i)) { top[k] = top[k - 1]; --k; }
    top[k] = Cand{a, v};
  }
  int head = 0;
  for (int k = 0; k < K; ++k) {
    heads[tid] = head < K ? top[head] : Cand{-INFINITY, 0x7fffffff};
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
      if (tid < w && better(heads[tid + w].v, heads[tid + w].i, heads[tid].v, heads[tid].i)) heads[tid] = heads[tid + w];
      __syncthreads();
    }
    const Cand best = heads[0];
    if (tid == 0) { cv[(long long)r * K + k] = best.v; ci[(long long)r * K + k] = best.i; }
    if (head < K && top[head].i == best.i && top[head].v == best.v) ++head;
    __syncthreads();
  }
}

struct MergeBufs {
  float* run_score; int* hist; int ld_hist; int* tab; int ld_tab; int* tok; int* parent;
  float* fin_score; int* fin_seq; int* fin_len; int* fin_flag; int* unsat;
  const float* row_lse; float* run_lse; float* fin_lse;      // null: no log-sum-exp tracking
};

// One block per clip.  Thread 0 runs the bookkeeping of _beam_search on the clip's beam * K candidates: the top 2 * beam by
// accumulated log-prob, the running beams (hits pushed down by 1e9), the finished set (length-normalised, merged with the
// earlier finished hypotheses, best beam kept) and the early-stop heuristic.  The block then gathers the new rows' token
// histories and slot tables from their parents, and copies finished sequences.  A clip whose heuristic has stopped it is
// left as it is: transformers keeps running its beams but can no longer change its finished set.  With row_lse, run_lse /
// fin_lse follow the hypotheses as their scores do: the sum over a hypothesis' steps of its processed rows' log-sum-exp.
__global__ void __launch_bounds__(128) merge_kernel(const float* __restrict__ cv, const int* __restrict__ ci, int beam, int K,
                                                    int V, int eot, int plen, int max_length, const int* __restrict__ gstep,
                                                    float length_penalty, MergeBufs B) {
  __shared__ int s_hist[kMaxBeam][kMaxLd];
  __shared__ int s_tab[kMaxBeam][kMaxLd];
  __shared__ int s_fin[kMaxBeam][kMaxLd];
  __shared__ int sel_par[kMaxBeam], sel_tok[kMaxBeam];
  __shared__ int fin_src[kMaxBeam], fin_tok[kMaxBeam], fin_len_new[kMaxBeam];     // src >= 0: old finished slot; < 0: -(row + 1)
  __shared__ int go;
  const int clip = blockIdx.x, tid = threadIdx.x, g = *gstep, cur = plen + g, r0 = clip * beam;
  if (tid == 0) go = B.unsat[clip];
  __syncthreads();
  if (!go) return;
  if (tid == 0) {
    const int NK = 2 * beam;
    float tv[2 * kMaxBeam]; int tf[2 * kMaxBeam];
    for (int k = 0; k < NK; ++k) { tv[k] = -INFINITY; tf[k] = 0x7fffffff; }
    for (int b = 0; b < beam; ++b)
      for (int k = 0; k < K; ++k) {
        const float v = cv[(long long)(r0 + b) * K + k];
        const int f = b * V + ci[(long long)(r0 + b) * K + k];
        if (!better(v, f, tv[NK - 1], tf[NK - 1])) continue;
        int q = NK - 1;
        while (q > 0 && better(v, f, tv[q - 1], tf[q - 1])) { tv[q] = tv[q - 1]; tf[q] = tf[q - 1]; --q; }
        tv[q] = v; tf[q] = f;
      }
    bool hit[2 * kMaxBeam]; float rv[2 * kMaxBeam];
    for (int k = 0; k < NK; ++k) {
      hit[k] = (tf[k] % V) == eot || cur + 1 >= max_length;
      rv[k] = tv[k] + (hit[k] ? -1.0e9f : 0.f);
    }
    // running beams: the best `beam` of rv, the lower candidate index first on a tie
    bool used[2 * kMaxBeam] = {};
    float nsc[kMaxBeam];
    for (int b = 0; b < beam; ++b) {
      int bi = -1;
      for (int k = 0; k < NK; ++k) if (!used[k] && (bi < 0 || rv[k] > rv[bi])) bi = k;
      used[bi] = true;
      sel_par[b] = tf[bi] / V; sel_tok[b] = tf[bi] % V; nsc[b] = rv[bi];
    }
    // finished hypotheses: the old set first, then the new candidates, best `beam` kept
    const float den = powf((float)(cur + 1 - plen), length_penalty);
    float ms[3 * kMaxBeam]; int msrc[3 * kMaxBeam], mtok[3 * kMaxBeam], mlen[3 * kMaxBeam], mdone[3 * kMaxBeam];
    float* fs = B.fin_score + (long long)clip * beam;
    const int* fl = B.fin_len + (long long)clip * beam;
    const int* fd = B.fin_flag + (long long)clip * beam;
    for (int j = 0; j < beam; ++j) { ms[j] = fs[j]; msrc[j] = j; mtok[j] = -1; mlen[j] = fl[j]; mdone[j] = fd[j]; }
    for (int k = 0; k < NK; ++k) {
      const bool did = hit[k] && k < beam;
      float v = tv[k] / den;
      v += did ? 0.f : -1.0e9f;
      ms[beam + k] = v; msrc[beam + k] = -(r0 + tf[k] / V + 1); mtok[beam + k] = tf[k] % V; mlen[beam + k] = g + 1;
      mdone[beam + k] = did;
    }
    bool mu[3 * kMaxBeam] = {};
    float nfs[kMaxBeam]; int nfd[kMaxBeam];
    for (int j = 0; j < beam; ++j) {
      int bi = -1;
      for (int k = 0; k < beam + NK; ++k) if (!mu[k] && (bi < 0 || ms[k] > ms[bi])) bi = k;
      mu[bi] = true;
      fin_src[j] = msrc[bi]; fin_tok[j] = mtok[bi]; fin_len_new[j] = mlen[bi]; nfs[j] = ms[bi]; nfd[j] = mdone[bi];
    }
    float mn = nfs[0];
    for (int j = 1; j < beam; ++j) mn = fminf(mn, nfs[j]);
    const float best_run = nsc[0] / powf((float)(cur + 1 - plen), length_penalty);
    bool any = false;
    for (int j = 0; j < beam; ++j) any |= best_run > (nfd[j] ? mn : -1.0e9f);
    for (int j = 0; j < beam; ++j) { fs[j] = nfs[j]; B.fin_flag[(long long)clip * beam + j] = nfd[j]; }
    for (int b = 0; b < beam; ++b) {
      B.run_score[r0 + b] = nsc[b];
      B.tok[r0 + b] = sel_tok[b];
      B.parent[r0 + b] = r0 + sel_par[b];
    }
    if (B.row_lse) {
      float nrl[kMaxBeam], nfl[kMaxBeam];
      for (int b = 0; b < beam; ++b) nrl[b] = B.run_lse[r0 + sel_par[b]] + B.row_lse[r0 + sel_par[b]];
      for (int j = 0; j < beam; ++j)
        nfl[j] = fin_src[j] >= 0 ? B.fin_lse[(long long)clip * beam + fin_src[j]] : B.run_lse[-fin_src[j] - 1] + B.row_lse[-fin_src[j] - 1];
      for (int b = 0; b < beam; ++b) B.run_lse[r0 + b] = nrl[b];
      for (int j = 0; j < beam; ++j) B.fin_lse[(long long)clip * beam + j] = nfl[j];
    }
    B.unsat[clip] = any ? 1 : 0;
  }
  __syncthreads();
  const int pos = cur - 1;                       // position of the token these logits were computed for
  for (int e = tid; e < beam * kMaxLd; e += blockDim.x) {
    const int b = e / kMaxLd, i = e - b * kMaxLd;
    const int pr = r0 + sel_par[b];
    if (i < g) s_hist[b][i] = B.hist[(long long)pr * B.ld_hist + i];
    if (i <= pos) s_tab[b][i] = B.tab[(long long)pr * B.ld_tab + i];
    const int src = fin_src[b];
    if (i < fin_len_new[b]) {
      if (src >= 0) s_fin[b][i] = B.fin_seq[((long long)clip * beam + src) * B.ld_hist + i];
      else s_fin[b][i] = i < g ? B.hist[(long long)(-src - 1) * B.ld_hist + i] : fin_tok[b];
    }
  }
  __syncthreads();
  for (int e = tid; e < beam * kMaxLd; e += blockDim.x) {
    const int b = e / kMaxLd, i = e - b * kMaxLd;
    if (i < g) B.hist[(long long)(r0 + b) * B.ld_hist + i] = s_hist[b][i];
    if (i == g) B.hist[(long long)(r0 + b) * B.ld_hist + i] = sel_tok[b];
    if (i <= pos) B.tab[(long long)(r0 + b) * B.ld_tab + i] = s_tab[b][i];
    if (i < fin_len_new[b]) B.fin_seq[((long long)clip * beam + b) * B.ld_hist + i] = s_fin[b][i];
    if (i == 0) B.fin_len[(long long)clip * beam + b] = fin_len_new[b];
  }
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_whisper_embed(const int32_t* tok, const float* emb, const float* pe, const int32_t* pos, int32_t R, int32_t d,
                                 float* x, evk_stream_t stream) {
  EVK_REQUIRE(tok && emb && pe && pos && x && R > 0 && d > 0, EVK_ERR_ARG, "whisper_embed: bad arguments");
  embed_kernel<<<R, 256, 0, (cudaStream_t)stream>>>(tok, emb, pe, pos, d, x);
  return check_launch("whisper_embed");
}

extern "C" int evk_whisper_add_pos(float* x, int64_t rows, int32_t T, int32_t d, const float* pe, evk_stream_t stream) {
  EVK_REQUIRE(x && pe && rows >= 0 && T > 0 && d > 0 && rows % T == 0, EVK_ERR_ARG, "whisper_add_pos: bad arguments");
  if (rows == 0) return EVK_OK;
  const long long blocks = (rows * d + 255) / 256;
  add_pos_kernel<<<(unsigned)(blocks < kNumSMs * 16 ? blocks : kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(x, rows, T, d, pe);
  return check_launch("whisper_add_pos");
}

extern "C" int evk_whisper_self_kv(const float* qkv, int32_t ldq, int32_t d, float* pool, int64_t ld_pool, int32_t* tab,
                                   int32_t ld_tab, const int32_t* pos, int32_t R, int32_t S, evk_stream_t stream) {
  EVK_REQUIRE(qkv && pool && tab && pos && R > 0 && d > 0 && ldq >= 3 * d && ld_pool >= 2 * d && S > 0 && S <= ld_tab, EVK_ERR_ARG,
              "whisper_self_kv: bad arguments");
  self_kv_kernel<<<R, 256, 0, (cudaStream_t)stream>>>(qkv, ldq, d, pool, ld_pool, tab, ld_tab, pos, S);
  return check_launch("whisper_self_kv");
}

extern "C" int evk_whisper_attn(const float* q, int32_t ldq, const float* kv, int64_t ld_kv, int32_t v_off, const int32_t* tab,
                                int32_t ld_tab, const int32_t* pos, int32_t n_keys, int32_t groups, int32_t nq, int32_t H,
                                float scale, float* o, int32_t ldo, evk_stream_t stream) {
  EVK_REQUIRE(q && kv && o && groups > 0 && H > 0 && nq >= 1 && nq <= kMaxBeam && ldq >= H * 64 && ldo >= H * 64, EVK_ERR_ARG,
              "whisper_attn: bad arguments");
  EVK_REQUIRE(tab ? (pos && nq == 1 && n_keys <= ld_tab) : n_keys > 0, EVK_ERR_ARG,
              "whisper_attn: slot-table mode takes one query per group and pos; cross mode takes n_keys > 0");
  EVK_REQUIRE(ld_kv % 4 == 0 && v_off % 4 == 0 && (uintptr_t)kv % 16 == 0, EVK_ERR_ARG, "whisper_attn: K rows must be 16-byte aligned");
  // slot-table mode sizes its score buffer for n_keys (the table width): *pos + 1 <= n_keys is the caller's contract
  const size_t smem = (size_t)nq * (64 + n_keys) * sizeof(float);
  EVK_REQUIRE(smem <= 200 * 1024, EVK_ERR_UNSUPPORTED, "whisper_attn: %d keys x %d queries exceed shared memory", n_keys, nq);
  static bool opted = false;
  if (!opted) {
    cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    opted = true;
  }
  attn_kernel<<<dim3(groups, H), 128, smem, (cudaStream_t)stream>>>(q, ldq, kv, ld_kv, v_off, tab, ld_tab, pos, n_keys, nq, scale, o, ldo);
  return check_launch("whisper_attn");
}

extern "C" int evk_whisper_layernorm(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, float* y,
                                     int32_t ldy, int64_t rows, int32_t C, evk_stream_t stream) {
  EVK_REQUIRE(x && gamma && beta && y && C > 0 && ldx >= C && ldy >= C && rows >= 0 && rows <= 0x7fffffff && x != y, EVK_ERR_ARG,
              "whisper_layernorm: bad arguments");
  if (rows == 0) return EVK_OK;
  row_layernorm_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(x, ldx, gamma, beta, eps, y, ldy, C);
  return check_launch("whisper_layernorm");
}

extern "C" int evk_whisper_first_pass(const float* logits, int64_t ld, int32_t R, int32_t V, int32_t nospeech,
                                      const int32_t* lang_ids, int32_t n_lang, float* nsp, int32_t* lang_tok, evk_stream_t stream) {
  EVK_REQUIRE(logits && lang_ids && nsp && lang_tok && R > 0 && V > 0 && n_lang > 0 && nospeech >= 0 && nospeech < V, EVK_ERR_ARG,
              "whisper_first_pass: bad arguments");
  first_pass_kernel<<<R, 512, 0, (cudaStream_t)stream>>>(logits, ld, V, nospeech, lang_ids, n_lang, nsp, lang_tok);
  return check_launch("whisper_first_pass");
}

extern "C" int evk_whisper_beam_step(const float* logits, int64_t ld, int32_t clips, int32_t beam, int32_t V, int32_t eot,
                                     int32_t nots, int32_t tsb, int32_t mit, int32_t plen, int32_t maxlen, const int32_t* sup,
                                     int32_t n_sup, const int32_t* bsup, int32_t n_bsup, const int32_t* gstep, float length_penalty,
                                     float* cand_val, int32_t* cand_tok, float* run_score, int32_t* hist, int32_t ld_hist,
                                     int32_t* tab, int32_t ld_tab, int32_t* tok, int32_t* parent, float* fin_score,
                                     int32_t* fin_seq, int32_t* fin_len, int32_t* fin_flag, int32_t* unsat, float* row_lse,
                                     float* run_lse, float* fin_lse, evk_stream_t stream) {
  EVK_REQUIRE(logits && gstep && cand_val && cand_tok && run_score && hist && tab && tok && parent && fin_score && fin_seq &&
              fin_len && fin_flag && unsat, EVK_ERR_ARG, "whisper_beam_step: null tensor");
  EVK_REQUIRE(!row_lse == !run_lse && !row_lse == !fin_lse, EVK_ERR_ARG,
              "whisper_beam_step: row_lse, run_lse and fin_lse are all given or all null");
  EVK_REQUIRE(clips > 0 && beam >= 1 && beam <= kMaxBeam && V > 0 && ld >= V && ld_hist <= kMaxLd && ld_tab <= kMaxLd &&
              (n_sup == 0 || sup) && (n_bsup == 0 || bsup), EVK_ERR_ARG, "whisper_beam_step: bad sizes clips=%d beam=%d V=%d", clips, beam, V);
  EVK_REQUIRE(eot >= 0 && eot < V && tsb > eot && tsb <= V && plen >= 1 && maxlen > plen && maxlen - plen <= ld_hist &&
              maxlen <= ld_tab, EVK_ERR_ARG, "whisper_beam_step: bad token layout or lengths");
  const int K = 2 * beam;
  StepCfg c{V, eot, nots, tsb, mit, sup, n_sup, bsup, n_bsup};
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)((V + 31) / 32) * sizeof(unsigned);
  EVK_REQUIRE(smem <= 32 * 1024, EVK_ERR_UNSUPPORTED, "whisper_beam_step: vocabulary of %d too large", V);
  cand_kernel<<<clips * beam, 512, smem, st>>>(logits, ld, c, hist, ld_hist, gstep, run_score, K, cand_val, cand_tok, row_lse);
  int rc = check_launch("whisper_beam_cand");
  if (rc) return rc;
  MergeBufs B{run_score, hist, ld_hist, tab, ld_tab, tok, parent, fin_score, fin_seq, fin_len, fin_flag, unsat, row_lse, run_lse, fin_lse};
  merge_kernel<<<clips, 128, 0, st>>>(cand_val, cand_tok, beam, K, V, eot, plen, maxlen, gstep, length_penalty, B);
  return check_launch("whisper_beam_merge");
}

extern "C" int evk_whisper_logmel(const float* wav, int64_t ld_wav, const int32_t* lens, int32_t B, int32_t T,
                                  const float* basis, const float* fb, int32_t n_mels, float* part, float* out,
                                  evk_stream_t stream) {
  EVK_REQUIRE(wav && lens && basis && fb && part && out, EVK_ERR_ARG, "whisper_logmel: null tensor");
  EVK_REQUIRE(B > 0 && B <= 65535 && T > 0 && n_mels > 0 && n_mels <= 256 && ld_wav >= kNfft / 2 + 1, EVK_ERR_ARG,
              "whisper_logmel: bad sizes B=%d T=%d n_mels=%d ld_wav=%lld", B, T, n_mels, (long long)ld_wav);
  cudaStream_t st = (cudaStream_t)stream;
  logmel_kernel<<<dim3((T + kFpb - 1) / kFpb, B), 256, 0, st>>>(wav, ld_wav, lens, basis, basis + kNfft * kBins, fb, n_mels, T, out);
  int rc = check_launch("whisper_logmel");
  if (rc) return rc;
  const int n_part = (T + kMaxChunk - 1) / kMaxChunk;
  logmel_max_kernel<<<dim3(n_part, B), 256, 0, st>>>(lens, n_mels, T, out, part);
  rc = check_launch("whisper_logmel_max");
  if (rc) return rc;
  const long long blocks = ((long long)T * n_mels + 256 * 16 - 1) / (256 * 16);
  logmel_norm_kernel<<<dim3((unsigned)blocks, B), 256, 0, st>>>(lens, n_mels, T, n_part, part, out);
  return check_launch("whisper_logmel_norm");
}

extern "C" int evk_whisper_window(const float* lm, int32_t B, int32_t T, int32_t n_mels, const int32_t* tab, int32_t R, float* out,
                                  evk_stream_t stream) {
  EVK_REQUIRE(lm && tab && out && B > 0 && T > 0 && n_mels > 0 && R > 0 && R <= 65535, EVK_ERR_ARG, "whisper_window: bad arguments");
  window_kernel<<<dim3((kFrames + kFpb - 1) / kFpb, R), 256, 0, (cudaStream_t)stream>>>(lm, T, n_mels, tab, out);
  return check_launch("whisper_window");
}
