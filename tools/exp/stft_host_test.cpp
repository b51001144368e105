// Host emulation of the STFT kernels' index arithmetic (csrc/stft_core.cuh) -- threads are a loop, barriers are phase
// boundaries.  Built as a shared object and driven from tests/test_cpu_stft_core.py against numpy and from
// tests/test_cpu_spectral_ref.py against the float64 error model, where stft_set_fault plants the modelled faults.
#include <cmath>
#include <vector>
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
#define EVK_HD static inline
#include "../../easevoice-trainer_b200/csrc/stft_core.cuh"
using namespace evk;

static std::vector<float2> g_tw;
static std::vector<float> g_hann;
static int g_fault_pass = -1, g_fault_win = 0;   // modelled faults: twiddle index + 1 in one pass; window read at j + 1
extern "C" void stft_set_fault(int pass, int win_shift) { g_fault_pass = pass; g_fault_win = win_shift; }
static void tables() {
  if (!g_tw.empty()) return;
  g_tw.resize(STFT_TAB + 1); g_hann.resize(STFT_TAB + 1);     // one entry of slack for the faults (the tables are periodic)
  for (int i = 0; i <= STFT_TAB; ++i) {
    const double a = 2.0 * M_PI * i / STFT_TAB;
    g_tw[i] = make_float2((float)std::cos(a), (float)(-std::sin(a)));
    g_hann[i] = (float)(0.5 - 0.5 * std::cos(a));
  }
}
static const float2* run_fft(int nt, int NH, float2* d0, float2* d1) {
  float2 *src = d0, *dst = d1;
  for (int Ns = 1, pass = 0; Ns < NH; ++pass) {
    int nn = Ns;
    const float2* tw = g_tw.data() + (pass == g_fault_pass ? 1 : 0);
    for (int tid = 0; tid < nt; ++tid) nn = stft_pass(tid, nt, NH, Ns, src, dst, tw);
    Ns = nn;
    float2* t = src; src = dst; dst = t;
  }
  return src;
}
extern "C" void stft_frame_fwd(const float* wav, int L, int s0, int N, int win, int nt, float* X /*[(N/2+1)*2]*/) {
  tables();
  const int NH = N / 2;
  std::vector<float2> d0(NH), d1(NH), sx(NH + 1);
  const float* hann = g_hann.data() + (g_fault_win ? STFT_TAB / win : 0);
  for (int tid = 0; tid < nt; ++tid) stft_load_phase(tid, nt, wav, L, s0, N, win, hann, d0.data());
  const float2* z = run_fft(nt, NH, d0.data(), d1.data());
  for (int tid = 0; tid < nt; ++tid) stft_untangle_phase(tid, nt, N, z, g_tw.data(), sx.data());
  for (int k = 0; k <= NH; ++k) { X[2 * k] = sx[k].x; X[2 * k + 1] = sx[k].y; }
}
// S[n] = sum_k Re(G[k] e^{+2 pi i k n / N})  (before the window factor)
extern "C" void stft_frame_adj(const float* G, int N, int nt, float* S) {
  tables();
  const int NH = N / 2;
  std::vector<float2> g(NH + 1), d0(NH), d1(NH);
  for (int k = 0; k <= NH; ++k) g[k] = make_float2(G[2 * k], G[2 * k + 1]);
  for (int tid = 0; tid < nt; ++tid) stft_adjoint_pack_phase(tid, nt, N, g.data(), g_tw.data(), d0.data());
  const float2* r = run_fft(nt, NH, d0.data(), d1.data());
  for (int m = 0; m < NH; ++m) { S[2 * m] = r[m].x; S[2 * m + 1] = -r[m].y; }
}
