// Bidirectional one-layer LSTM recurrence (torch.nn.LSTM semantics: gate order i, f, g, o, zero initial h and c),
// inference only.  It runs the LSTMModule of the UVR5 DeEcho / DeReverb CascadedNet (uvr5.py) over the frame axis.
//
// The caller has already added the input projections of both directions, biases included (one GEMM):
//   G(t, n) = [x(t, n) . W_ih_fwd^T + b_fwd | x(t, n) . W_ih_rev^T + b_rev]          8H floats, [direction][gate][H]
// and this kernel runs  gates = G(t, n)[d] + W_hh_d . h_{t -/+ 1},  c = f c + i g,  h = o tanh(c)  for all T steps,
// writing y(t, n) = [h_fwd(t) | h_rev(t)]  (2H floats, the nn.LSTM output layout).
//
// One persistent launch: CTA = one direction x up to 4 batch rows, 4H threads.  Thread (u, q) keeps in registers the four
// gate rows of hidden unit u of W_hh restricted to its quarter q of the contraction (k = 16 v + 4 q + e), reads h from
// shared memory as float4s, and the four quarters are summed with two butterfly shuffles, so every lane of the quad holds
// the four gate pre-activations of (u, row).  Lane q then updates the cell of row q: c stays in a register, the new h goes
// to the other half of a double-buffered shared array, and one __syncthreads() per step orders the steps.  The next
// step's G values are loaded before the current step's contraction.
//
// Exact fp32 FMAs and the accurate expf / tanhf.  A row's arithmetic does not depend on which other rows share its CTA or
// the launch, and there are no atomics: results are bit-reproducible and independent of the batch.
#include "evk_common.cuh"

namespace evk {
namespace {

constexpr int MAX_ROWS = 4;           // batch rows per CTA: one cell-updating lane per row in each quad

struct LstmArgs {
  const float* g; long long g_st, g_sn;
  const float* w;
  float* y; long long y_st, y_sn;
  int T, N, rows;
};

__device__ __forceinline__ float sigmoid_f(float v) { return 1.f / (1.f + expf(-v)); }

template <int H>
__global__ void __launch_bounds__(4 * H) lstm_bidir_kernel(LstmArgs a) {
  constexpr int KL = H / 4;            // contraction elements per thread
  constexpr int NV = KL / 4;           // float4s of h per thread and row
  __shared__ __align__(16) float hs[2][MAX_ROWS][H];
  const int tid = threadIdx.x, q = tid & 3, u = tid >> 2;
  const int d = blockIdx.x & 1, n0 = (blockIdx.x >> 1) * a.rows;
  const int R = min(a.rows, a.N - n0);

  float w[4][KL];
  const float* wd = a.w + (long long)d * 4 * H * H;
#pragma unroll
  for (int gt = 0; gt < 4; ++gt)
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int e = 0; e < 4; ++e) w[gt][4 * v + e] = __ldg(wd + (long long)(gt * H + u) * H + 16 * v + 4 * q + e);
  for (int i = tid; i < MAX_ROWS * H; i += 4 * H) (&hs[0][0][0])[i] = 0.f;

  const bool cell = q < R;             // lane q of the quad updates row n0 + q
  const int dt = d ? -1 : 1;
  int t = d ? a.T - 1 : 0;
  const float* gp = a.g + (cell ? (long long)(n0 + q) * a.g_sn : 0) + d * 4 * H + u;
  float* yp = a.y + (cell ? (long long)(n0 + q) * a.y_sn : 0) + d * H + u;
  float gx[4] = {0.f, 0.f, 0.f, 0.f}, c = 0.f;
  if (cell) {
#pragma unroll
    for (int gt = 0; gt < 4; ++gt) gx[gt] = __ldg(gp + t * a.g_st + gt * H);
  }
  __syncthreads();

  for (int s = 0; s < a.T; ++s, t += dt) {
    float gn[4] = {0.f, 0.f, 0.f, 0.f};
    if (cell && s + 1 < a.T) {
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) gn[gt] = __ldg(gp + (t + dt) * a.g_st + gt * H);
    }
    const float* hc = &hs[s & 1][0][0];
    float mine[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < R; ++r) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      const float4* hp = reinterpret_cast<const float4*>(hc + r * H) + q;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const float4 h4 = hp[4 * v];
#pragma unroll
        for (int gt = 0; gt < 4; ++gt) {
          acc[gt] = fmaf(w[gt][4 * v + 0], h4.x, acc[gt]);
          acc[gt] = fmaf(w[gt][4 * v + 1], h4.y, acc[gt]);
          acc[gt] = fmaf(w[gt][4 * v + 2], h4.z, acc[gt]);
          acc[gt] = fmaf(w[gt][4 * v + 3], h4.w, acc[gt]);
        }
      }
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) {     // a + b == b + a in fp32: the four lanes of the quad end with the same bits
        acc[gt] += __shfl_xor_sync(0xffffffffu, acc[gt], 1);
        acc[gt] += __shfl_xor_sync(0xffffffffu, acc[gt], 2);
      }
      if (r == q) {
#pragma unroll
        for (int gt = 0; gt < 4; ++gt) mine[gt] = acc[gt];
      }
    }
    if (cell) {
      const float ig = sigmoid_f(gx[0] + mine[0]), fg = sigmoid_f(gx[1] + mine[1]);
      const float gg = tanhf(gx[2] + mine[2]), og = sigmoid_f(gx[3] + mine[3]);
      c = fmaf(fg, c, ig * gg);
      const float h = og * tanhf(c);
      hs[(s + 1) & 1][q][u] = h;
      yp[t * a.y_st] = h;
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) gx[gt] = gn[gt];
    }
    __syncthreads();                   // h_t complete; every read of the other buffer is done
  }
}

template <int H>
int launch_lstm(const LstmArgs& a, cudaStream_t st) {
  const int grid = 2 * cdiv(a.N, a.rows);
  lstm_bidir_kernel<H><<<grid, 4 * H, 0, st>>>(a);
  return check_launch("lstm_bidir_fwd");
}

}  // namespace
}  // namespace evk

using namespace evk;

extern "C" int evk_lstm_bidir_fwd(const float* g, int64_t g_st, int64_t g_sn, const float* w_hh, float* y, int64_t y_st,
                                  int64_t y_sn, int32_t T, int32_t N, int32_t H, cudaStream_t st) {
  EVK_REQUIRE(g && w_hh && y, EVK_ERR_ARG, "lstm_bidir_fwd: null tensor");
  EVK_REQUIRE(H == 32 || H == 64, EVK_ERR_ARG, "lstm_bidir_fwd: hidden size %d not supported (32 or 64)", H);
  EVK_REQUIRE(T > 0 && N > 0, EVK_ERR_ARG, "lstm_bidir_fwd: bad sizes T=%d N=%d", T, N);
  EVK_REQUIRE(g_st >= 0 && g_sn >= 0 && y_st >= 0 && y_sn >= 0, EVK_ERR_ARG, "lstm_bidir_fwd: negative stride");
  // rows per CTA: one row (2N CTAs, two per SM) up to N = 132, then up to 4 rows, so the grid stays near one wave
  int rows = cdiv(N, kNumSMs);
  if (rows > MAX_ROWS) rows = MAX_ROWS;
  LstmArgs a{g, g_st, g_sn, w_hh, y, y_st, y_sn, T, N, rows};
  if (H == 32) return launch_lstm<32>(a, st);
  return launch_lstm<64>(a, st);
}
