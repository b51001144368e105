/* libevk_sm90.so -- C ABI of the H100-native EaseVoice stage-2 hot path.
 *
 * The reference (megaease/easevoice-trainer) is pure Python on stock PyTorch: it has NO operator /
 * FFI interface.  Every entry point below therefore replaces a *call site* of the reference that
 * lowers to a library kernel; the citation after each declaration is that call site
 * (paths relative to the reference's src/easevoice/module unless noted).  INTEGRATION.md shows the
 * ctypes binding a reference maintainer would add.
 *
 * Conventions
 *  - All pointers are raw DEVICE pointers owned by the caller (PyTorch); the library never
 *    allocates, frees or retains them.  Sizes/strides are explicit, in ELEMENTS.
 *  - Activations are channels-last: a [B, T, C] tensor is B*T rows of C floats with row pitch `ld`.
 *  - All work is enqueued on `stream`; no hidden synchronisation, no default-stream use; every
 *    entry point is CUDA-graph capturable.  Returns 0 or a negative evk_status;
 *    evk_last_error() gives the thread-local message.  Never throws, never exits.
 *  - sm_90a only: evk_init() fails on any other device.  There is no CPU fallback.
 */
#ifndef EVK_H_
#define EVK_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* evk_stream_t;

enum evk_status { EVK_OK = 0, EVK_ERR_ARG = -1, EVK_ERR_CUDA = -2, EVK_ERR_ARCH = -3, EVK_ERR_UNSUPPORTED = -4 };
/* EVK_ACT_GELU: exact erf form, x * 0.5 * (1 + erf(x / sqrt(2))) (nn.GELU()); forward epilogues only. */
enum evk_act { EVK_ACT_NONE = 0, EVK_ACT_LRELU = 1, EVK_ACT_RELU = 2, EVK_ACT_TANH = 3, EVK_ACT_GELU = 4 };

#define EVK_MAX_TAPS 48

int evk_init(void);                    /* checks compute capability 9.0, raises smem limits */
int evk_version(void);
const char* evk_last_error(void);
int evk_sync_check(evk_stream_t stream); /* cudaStreamSynchronize + error fetch (tests only) */

/* ------------------------------------------------------------------------------------------
 * Generalised 1-D convolution as a tap-sum of GEMMs (tensor cores, TF32 in / FP32 accumulate)
 *
 *   Y[z][(o0 + j*os)*P + w][n] = epi( sum_{q<Q} sum_{c<C} X[z][(j*is + off[q])*P + w][c] * W[z][q][n][c] )
 *
 * for j in [0,J), w in [0,P); input rows outside [0, Tin*P) (or >= in_len[b]*P) read as zero.
 * z = b*H + h addresses a two-level batch (X + b*x_sb + h*x_sh, same for W/Y/R; w_sb = w_sh = 0
 * shares one weight).  epi(v) = mask(act(v + bias[n] + R[...][n])) with mask = (row/P < out_len[b]).
 * Covers: Conv1d / Conv2d(k,1) forward (models.py:452-471,538-587; modules.py:187-212,298-311;
 * attentions.py:408-416), their data gradients (evk_gconv_dgrad), ConvTranspose1d (models.py:460; the data gradient of
 * a conv), nn.Linear / 1x1 convs, and the attention GEMMs (attentions.py:243-292).
 * ------------------------------------------------------------------------------------------ */
typedef struct evk_gconv_desc {
  const float* x; float* w; float* y; const float* res; const float* bias;
  const int32_t* in_len; const int32_t* out_len;
  int64_t x_sb, x_sh, w_sb, w_sh, w_sq, y_sb, y_sh, r_sb, r_sh;
  int32_t ldx, ldw, ldy, ldr;
  int32_t b_sh;          /* bias offset per inner-batch index h */
  int32_t Z, H;          /* batch count and inner (head) count: b = z / H, h = z % H */
  int32_t C, N, Q, G;    /* in-channels, out-channels, taps, groups (G > 1: W is [Q][N][C/G]) */
  int32_t Tin, J, P;     /* input positions per batch, output positions computed, inner width */
  int32_t is, os, o0;    /* input stride, output stride, output origin (in positions) */
  int32_t Tout;          /* output positions per batch (bounds for (o0 + j*os)) */
  int32_t act; float slope;
  int32_t off[EVK_MAX_TAPS];
  /* optional dropout AFTER the activation, forward only: y = mask(dropout_p(act(...))); rng = device [seed, offset] (the
   * library's RNG state), sid = stream id; active when drop_rng && drop_p > 0, and then act must be EVK_ACT_RELU (EVK_ERR_ARG
   * otherwise: a backward recovers the mask from the saved output).  The output at element offset e from y is kept (scaled
   * by 1/(1-p)) or dropped by dropk_scale4(e / 4)[e % 4] (csrc/evk_common.cuh), whatever route serves the launch: routes 1
   * and 2 apply it in gemm_tma_kernel's epilogue, every other route in one in-place pass over y after the launch. */
  const uint64_t* drop_rng; uint64_t drop_sid; float drop_p;
  /* 1: not route 1 of evk_gconv_fwd.  ConvTranspose1d's data gradient, which has always run on gconv_f_kernel: route 1
   * would take it for the HiFi-GAN generator's stride-2 upsampling layers (128 -> 64, 64 -> 32) and change their bits. */
  int32_t no_phase_split;
  /* 1: the caller takes no gradient through this launch, so route 0 of evk_gconv_fwd may serve it exactly in fp32. */
  int32_t no_grad;
} evk_gconv_desc;

/* Any stride and alignment; groups as G.  Routes, the first that takes the launch runs it:
 *   0. no_grad, a Linear of 1 <= Z*J*P <= 4 dense rows (Q == 1, off[0] == 0, is == os == 1, o0 == 0, J <= Tin, G <= 1,
 *      H == 1, x_sb == J*P*ldx and y_sb == J*P*ldy unless Z == 1), no res, in_len, out_len or dropout, act NONE / RELU /
 *      LRELU, 4 <= C <= ldw, C % 4 == 0, ldw % 4 == 0, w 16-byte aligned, ldx >= C, ldy >= N, within evk_gemv_rows'
 *      staging limit: evk_gemv_rows, exact fp32 (the rule is gconv_fwd_gemv in csrc/gemv_route.h);
 *   1. 1 < is <= 4, no_phase_split == 0, G <= 1, H == 1, no in_len, C % 4 == 0, C, N >= 32, Z*J*P >= 2048, J*P >= 64:
 *      x split into `is` phase copies (library scratch), then a stride-1 tap sum over them on gemm_tma_kernel;
 *   2. stride 1 on gemm_tma_kernel (shape rule in gemm_tma_plan);  3. stride 1 on gconv_tc_kernel;  4. gconv_f_kernel;
 *   5. the direct kernel when X or W is not 16-byte tileable (x, w 16-byte aligned, ldx, ldw and strides multiples of 4).
 * Routes 2-4 run groups as the inner batch.  Precise mode skips 1-3, evk_set_backend(0) 2-3, evk_set_backend_tma(0) 1-2.
 * Route 1 checks all of gemm_tma_kernel's conditions before it splits x. */
int evk_gconv_fwd(const evk_gconv_desc* d, evk_stream_t stream);
int evk_gconv_desc_size(void);         /* sizeof(evk_gconv_desc) as compiled: bindings check their mirror against it */
/* 0 (default): one TF32 product per MAC.  1: 3xTF32 error-compensated products (~fp32 accuracy, 3x tensor work);
 * the parity tests use it to separate indexing errors from TF32 operand rounding. Process-wide. */
int evk_set_precise(int32_t on);
int evk_get_precise(void);
/* 1 (default): eligible stride-1 launches run on the wgmma kernels (gemm_tma.cu, gconv_tc.cu); 0: on mma.sync. */
int evk_set_backend(int32_t tensor_core);
/* Dispatch accounting: algorithmic flops enqueued since the last reset, per kernel family (host-side counters; graph
 * replays add nothing).  out[i], i < EVK_DISPATCH_SLOTS:
 *   0 conv/linear fwd-like on gemm_tma_kernel (TMA + wgmma)   1 ... on gconv_tc_kernel (wgmma, staged slab)
 *   2 ... on gconv_f_kernel (mma.sync)                          3 ... on the direct CUDA-core kernels
 *   4 weight gradients on gemm_tma_kernel                        5 ... on gconv_w_kernel (mma.sync)
 *   6 ... on the direct kernels                                  7 plain evk_gemm_tf32 calls
 *   8 conv/linear fwd-like on evk_gemv_rows (route 0 of evk_gconv_fwd) */
/* A/B switches of gemm_tma_kernel: slab (default 1) = stride-1 tap sums stage one input slab per channel block and run every
 * tap from it; mt2 (default 1) = 256-row tiles where the persistent grid's wave quantisation allows; trunc_comp (default
 * 3.52e-4) = accumulator compensation per raw fp32 operand for the tensor core's TF32 operand truncation (0 disables). */
int evk_set_tma_options(int32_t slab, int32_t mt2, float trunc_comp);
#define EVK_DISPATCH_SLOTS 9
int evk_dispatch_stats(double* out, int32_t n);
int evk_dispatch_stats_reset(void);
/* Weight gradient of the same operator:  W[z][q][n][c] += sum_{j,w} Yg[z][orow][n] * X[z][irow][c]
 * (d->y is read as the output gradient, d->w is accumulated -- partial sums added in a fixed order, so the result is
 * reproducible; when w_sb == w_sh == 0 the sum also runs over z).  Replaces autograd's conv weight-gradient kernels for the
 * call sites above.  dyt (nullable) [Z][N][ld_dyt] = Yg transposed (evk_dy_prep).  Routes:
 *   1. dyt given and evk_gconv_wgrad_takes_dyt: conv_wgrad_kernel, per stride phase's taps on phase copies of X (scratch),
 *      K split in max(1, min(64, SMs / tiles, Z * ceil(J*P / 32) / 8)), tiles = taps * ceil(N / 128) * ceil(C / 128);
 *   2. gconv_w_kernel, groups as the inner batch;  3. the direct kernel when X or Yg is not 16-byte tileable. */
int evk_gconv_wgrad(const evk_gconv_desc* d, const float* dyt, int32_t ld_dyt, evk_stream_t stream);
/* 1 when evk_gconv_wgrad takes route 1 given dyt (callers ask evk_dy_prep for dyt only then): is <= 4 (taps at consecutive
 * offsets when strided: any dilation when Q == 1), G <= 1, H == 1, os == 1, o0 == 0, w_sb == 0, no in_len, C % 4 == 0,
 * C, N >= 32, Z*J*P >= 2048, J*P >= 64, X and Yg 16-byte tileable, not precise. */
int evk_gconv_wgrad_takes_dyt(const evk_gconv_desc* d);
/* Data gradient of the conv that d describes as evk_gconv_fwd takes it (is = stride, off[q] = q*dil - pad, W = PA
 * [Q][N][C/G]), with the roles of x and y swapped: d->y is dY [Z][J*P][N] and is read, d->x is dX and is written, a dense
 * [Z][Tin*P][C] tensor (ldx == C; H == 1).  wt (nullable) is the transposed weight PB [Q][C/G][ld_wt].  d->bias
 * (nullable) is added to every row of dX: ConvTranspose1d's forward is this call.  Routes:
 *   1. wt 16-byte tileable (ld_wt % 4 == 0, 16-byte aligned), dY too (ldy, y_sb multiples of 4, 16-byte aligned) and,
 *      when G > 1, C/G and N/G multiples of 4: the polyphase plan (csrc/dgrad_plan.h), one stride-1 launch of routes
 *      2-4 of evk_gconv_fwd per residue of the taps mod is, each writing every is-th row of dX: dY as the input, PB
 *      offset by q0 taps with an is-fold tap pitch as the weight, os = is, o0 = the phase's first row, groups as the
 *      inner batch.  A strided conv needs taps at consecutive offsets (dilation 1).  When Q < is, dX is zeroed first
 *      (rows of a residue with no tap stay zero, without the bias);
 *   2. otherwise the direct kernel.
 * With d->in_len, rows t*P + w of dX with t >= in_len[b] are zeroed afterwards: the forward read them as zero.
 * With d->out_len (it bounds dX, the rows this call writes, not the forward's output), rows t*P + w of dX with
 * t >= out_len[b] are written as zero: by the epilogues of route 1's launches (the length mask of evk_gconv_fwd), after
 * route 2.  ConvTranspose1d over rows of different lengths passes its output lengths here; its input rows past a row's
 * length must hold zeros, which they do when they come from launches masked the same way. */
int evk_gconv_dgrad(const evk_gconv_desc* d, const float* wt, int32_t ld_wt, evk_stream_t stream);

/* out[n] (+)= sum_rows x[row][n]  -- bias gradients */
int evk_colsum(const float* x, int64_t rows, int32_t n, int32_t ld, float* out, int32_t accumulate, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Weight preparation: torch.nn.utils.weight_norm (modules.py:154-171, models.py:425-435,489-587)
 * folded into the operand-packing pass (pack.cu).  One job: v is [D0][D1][Q] (torch layout), g is [D0] or NULL (plain
 * weight).  Produces PA[q][d0][d1] ([Q][D0p][lda]) and, unless pb is NULL, PB[q][d1][d0] ([Q][D1p][ldb]); D0p x D1p
 * zero-pad the channel dims (padding pre-zeroed by the caller) so 1-channel layers run on the tensor-core kernels.
 * The backward takes dPA (gradient in PA layout) and writes dv [D0][D1][Q] and dg [D0] (when g is not NULL).
 * ------------------------------------------------------------------------------------------ */
typedef struct evk_pack_job {
  const float* v; const float* g; float* pa; float* pb;
  const float* dpa; float* dv; float* dg;             /* backward only */
  int32_t D0, D1, Q, lda, D0p, ldb, D1p, row0;        /* row0: the job's first row (block) in a table; 0 for one job */
} evk_pack_job;
int evk_pack_job_size(void);           /* sizeof(evk_pack_job) as compiled: bindings check their mirror against it */
int evk_weight_pack_one(const evk_pack_job* j, evk_stream_t stream);       /* one weight; *j is read on the host */
int evk_weight_pack_bwd_one(const evk_pack_job* j, evk_stream_t stream);
/* A whole network per launch: `jobs` is a DEVICE array, job_of_row [nrows] maps each (job, output-channel) row to its job. */
int evk_weight_pack_batched(const evk_pack_job* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream);
int evk_weight_pack_bwd_batched(const evk_pack_job* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused mel front end (mel_processing.py:40-142): reflect-pad -> Hann -> rFFT(2048) ->
 * sqrt(re^2+im^2+1e-6) -> sparse Slaney filterbank -> log(clamp 1e-5).
 * wav [B][L] (pitch ldw); outputs channels-last: spec [B*T][n_fft/2+1] (pitch ld_spec, nullable),
 * mel [B*T][n_mels] (pitch ld_mel, nullable), cplx [B*T][n_fft/2+1][2] (nullable, saved for bwd).
 * Filterbank is CSR by mel row: fb_ptr[n_mels+1], fb_idx[nnz], fb_val[nnz].
 * lens (nullable, int32 [B]): per-row valid length; the reflection sits at each row's own end and frames past the row's
 * own count are written as zeros / log(1e-5) (what the reference's per-utterance features + zero-padding collate give).
 * ------------------------------------------------------------------------------------------ */
int evk_mel_fwd(const float* wav, const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t hop, int32_t n_mels,
                const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val, float* spec, int32_t ld_spec,
                float* mel, int32_t ld_mel, float* cplx, evk_stream_t stream);
/* 1 (default): warp-per-frame register FFT; 0: the general block-per-frame kernel (evk_stft_fwd), kept for A/B parity. */
int evk_set_mel_variant(int32_t v);
/* gradient wrt wav of sum(dmel * mel): dwav [B][L] must be zero-initialised (overlap-add). */
int evk_mel_bwd(const float* dmel, int32_t ld_dmel, const float* cplx, const float* mel, int32_t ld_mel, const int32_t* lens,
                int32_t B, int32_t L, int32_t ldw, int32_t hop, int32_t n_mels, const int32_t* fb_ptr, const int32_t* fb_idx,
                const float* fb_val, float* dwav, evk_stream_t stream);
/* General STFT (stft.cu): n_fft in {256..8192} (power of two), any hop, power-of-two win <= n_fft (periodic Hann, centred in
 * the frame as torch.stft does), reflect padding `pad` on both sides, T frames per row starting at f*hop - pad:
 *   mel_processing.py:40-74  -> pad = (n_fft - hop) / 2, T = (L + 2 pad - n_fft) / hop + 1
 *   torch.stft(center=True)  -> pad = n_fft / 2,         T = 1 + L / hop        (bs_roformer.py:565-581, the MR-STFT loss)
 * Outputs (each nullable): cplx [B*T][n_fft/2+1][2]; spec [B*T][ld_spec] = sqrt(re^2+im^2+mag_eps); mel [B*T][ld_mel] =
 * log(max(fb . spec, clip)), filterbank in CSR-by-mel form. */
int evk_stft_fwd(const float* wav, const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t n_fft, int32_t hop, int32_t win,
                 int32_t pad, int32_t T, float mag_eps, float* cplx, float* spec, int32_t ld_spec, int32_t n_mels,
                 const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val, float clip, float* mel, int32_t ld_mel,
                 evk_stream_t stream);
/* Adjoint: dwav [B][ldw] (zero-initialised by the caller) += d/dwav, from either gcplx [B*T][n_fft/2+1][2] (dL/dRe, dL/dIm) or,
 * when gcplx is null, from dmel with the forward's saved cplx and mel. */
int evk_stft_bwd(const float* gcplx, const float* dmel, int32_t ld_dmel, const float* cplx, const float* mel, int32_t ld_mel,
                 float mag_eps, float clip, int32_t n_mels, const int32_t* fb_ptr, const int32_t* fb_idx, const float* fb_val,
                 const int32_t* lens, int32_t B, int32_t L, int32_t ldw, int32_t n_fft, int32_t hop, int32_t win, int32_t pad,
                 int32_t T, float* dwav, evk_stream_t stream);
/* loss[0] += scale * sum_i |a_i - b_i| over n complex elements (F.l1_loss on complex tensors); grad (nullable, [n][2]) =
 * scale * (a - b) / |a - b|. */
int evk_cplx_l1(const float* a, const float* b, int64_t n, float scale, float* loss, float* grad, evk_stream_t stream);
/* spec_to_mel_torch (mel_processing.py:77-90): spec [rows][F] -> log-mel [rows][n_mels] */
int evk_spec_to_mel(const float* spec, int64_t rows, int32_t ld_spec, int32_t n_mels, const int32_t* fb_ptr,
                    const int32_t* fb_idx, const float* fb_val, float* mel, int32_t ld_mel, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Element-wise / row-wise kernels (all tensors are [rows][C] views with explicit pitches)
 * ------------------------------------------------------------------------------------------ */
/* generic unary map y = f(x); op: 0 copy*alpha, 1 lrelu(alpha), 2 tanh, 3 mish, 4 relu, 6 gelu (exact erf form, forward only).
 * bwd: dx = dy*f'(x) (op 5 there: tanh with the derivative taken from the saved OUTPUT) */
/* GroupNorm with one channel per group over the time axis of a channels-last tensor (torch.nn.GroupNorm(C, C) of the HuBERT
 * feature extractor, transformers modeling_hubert.py HubertGroupNormConvLayer): y[b][t][c] = (x - mean_t) * rsqrt(var_t + eps)
 * * gamma[c] + beta[c], biased variance; optional exact GELU applied to the result (act_gelu != 0).  Forward only.
 * lens (nullable, int32 device [B]): mean and variance of item b over t < lens[b] only, frames t >= lens[b] written as 0; a
 * fixed summation order (no atomics), so an item's result does not depend on T or on the padding.  NULL: every frame. */
int evk_instnorm_cl(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, int32_t act_gelu, float* y,
                    int32_t ldy, int32_t B, int32_t T, int32_t C, const int32_t* lens, evk_stream_t stream);
/* evk_instnorm_cl without lens for large planes (nn.InstanceNorm2d(affine=True) over the T = H * W pixels of a channels-last
 * [B, H, W, C] operand, the MDX23C U-Net's norm before every conv and Linear): the same shifted sums, split over chunks of
 * 2048 pixels whose partials are added in chunk order (no atomics; an item's result does not depend on B), then one
 * element-wise pass that normalises (+ exact GELU).  Item b's pixels start at x + b T ldx. */
int evk_instnorm_plane(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, int32_t act_gelu,
                       float* y, int32_t ldy, int32_t B, int64_t T, int32_t C, evk_stream_t stream);
int evk_unary(int32_t op, float alpha, const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows, int32_t C,
              evk_stream_t stream);
int evk_unary_bwd(int32_t op, float alpha, const float* x, int32_t ldx, const float* dy, int32_t lddy, float* dx,
                  int32_t lddx, int64_t rows, int32_t C, evk_stream_t stream);
/* y = alpha*a + beta*b (+ gamma*c), optional row mask (t < len[b], T rows per batch); b,c nullable */
int evk_axpby(const float* a, int32_t lda, float alpha, const float* b, int32_t ldb, float beta, const float* c,
              int32_t ldc, float gamma, float* y, int32_t ldy, int64_t rows, int32_t C, const int32_t* len,
              int32_t T, evk_stream_t stream);
/* y[b][t][:] = x[b][t][:] + v[b][:]   (models.py:454 `x + self.cond(g)`) */
int evk_add_bvec(const float* x, int32_t ldx, const float* v, int32_t ldv, float* y, int32_t ldy, int32_t B,
                 int32_t T, int32_t C, evk_stream_t stream);
/* WaveNet gate (commons.py:94-101): acts = tanh(a[:, :H] + g[b][:H]) * sigmoid(a[:, H:] + g[b][H:]) */
int evk_wn_gate(const float* a, int32_t lda, const float* g, int32_t ldg, float* acts, int32_t ldo, int32_t B,
                int32_t T, int32_t Hc, evk_stream_t stream);
int evk_wn_gate_bwd(const float* a, int32_t lda, const float* g, int32_t ldg, const float* dacts, int32_t lddo,
                    float* da, int32_t ldda, int32_t B, int32_t T, int32_t Hc, evk_stream_t stream);
/* GLU with residual (modules.py:553-559): y = x + h[:, :C] * sigmoid(h[:, C:])  (x nullable => plain GLU) */
int evk_glu_res(const float* x, int32_t ldx, const float* h, int32_t ldh, float* y, int32_t ldy, int64_t rows,
                int32_t C, evk_stream_t stream);
int evk_glu_res_bwd(const float* h, int32_t ldh, const float* dy, int32_t lddy, float* dh, int32_t lddh, int64_t rows,
                    int32_t C, evk_stream_t stream);
/* posterior reparameterisation (models.py:357-358): z = (m + noise*exp(logs)) * mask */
int evk_reparam(const float* stats, int32_t lds, const float* noise, int32_t ldn, float* z, int32_t ldz, int32_t B,
                int32_t T, int32_t C, const int32_t* len, evk_stream_t stream);
int evk_reparam_bwd(const float* stats, int32_t lds, const float* noise, int32_t ldn, const float* dz, int32_t lddz,
                    float* dstats, int32_t ldds, int32_t B, int32_t T, int32_t C, const int32_t* len,
                    evk_stream_t stream);
/* row mask: y = x * (t < len[b]) */
int evk_rowmask(const float* x, int32_t ldx, float* y, int32_t ldy, int32_t B, int32_t T, int32_t C,
                const int32_t* len, evk_stream_t stream);
/* channel reversal (modules.py:376-383 Flip): y[r][c] = x[r][C-1-c] */
int evk_flip_channels(const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows, int32_t C,
                      evk_stream_t stream);
/* segment gather (commons.py:42-48): y[b][j][:] = x[b][ids[b]*mul + j][:]; bwd scatters into zeroed dx */
int evk_slice_rows(const float* x, int32_t ldx, int32_t Tin, const int64_t* ids, int32_t mul, float* y, int32_t ldy,
                   int32_t B, int32_t seg, int32_t C, int32_t scatter, evk_stream_t stream);
/* right reflect pad of a [B][T] 1-channel signal to Tp (models.py:543-546); bwd folds */
int evk_reflect_pad_right(const float* x, int32_t T, float* y, int32_t Tp, int32_t B, int32_t bwd,
                          evk_stream_t stream);
/* layout change at the API boundary: [B][C][T] <-> [B][T][C(ld)] */
int evk_transpose_bct_btc(const float* x, float* y, int32_t B, int32_t C, int32_t T, int32_t ld, int32_t to_btc,
                          evk_stream_t stream);
/* embedding gather y[r][:] = table[idx[r / rep]][:]  (rep=2: models.py:924-927 nearest x2) and its
 * scatter-add gradient (rep must be 1).  rows == 0 is a no-op (the pointers of an empty tensor may then be null). */
int evk_embedding(const float* table, int32_t ldt, const int64_t* idx, int64_t rows, int32_t rep, float* y,
                  int32_t ldy, int32_t C, evk_stream_t stream);
/* dtable[idx[r]][c] += dy[r][c] for the V-row table; every entry sums its rows in row order (reproducible). */
int evk_embedding_bwd(const float* dy, int32_t lddy, const int64_t* idx, int64_t rows, float* dtable, int32_t ldt,
                      int32_t C, int32_t V, evk_stream_t stream);
/* masked temporal mean (modules.py:729-737): y[b][:] = sum_{t<len[b]} x[b][t][:] / len[b]; bwd broadcast */
int evk_masked_mean(const float* x, int32_t ldx, float* y, int32_t ldy, int32_t B, int32_t T, int32_t C,
                    const int32_t* len, int32_t bwd, evk_stream_t stream);
/* inverted dropout with a Philox stream; seed/offset live in device memory (graph replay safe) */
int evk_dropout(const float* x, float* y, int64_t n, float p, const uint64_t* seed_offset, uint64_t stream_id,
                evk_stream_t stream);
/* standard normal noise (models.py:358 randn_like) and uniform slice ids (commons.py:51-58) */
int evk_randn(float* y, int64_t n, const uint64_t* seed_offset, uint64_t stream_id, evk_stream_t stream);
int evk_rand_slice_ids(int64_t* ids, const int32_t* len, int32_t B, int32_t seg, const uint64_t* seed_offset,
                       uint64_t stream_id, evk_stream_t stream);
int evk_advance_rng(uint64_t* seed_offset, uint64_t inc, evk_stream_t stream);

/* channel LayerNorm (modules.py:28-31) over the C floats of each row; saves mean/rstd [rows][2] */
int evk_layernorm_fwd(const float* x, int32_t ldx, const float* res, int32_t ldr, const float* gamma,
                      const float* beta, float eps, float* y, int32_t ldy, float* stats, int64_t rows, int32_t C,
                      evk_stream_t stream);
int evk_layernorm_bwd(const float* x, int32_t ldx, const float* res, int32_t ldr, const float* gamma,
                      const float* stats, const float* dy, int32_t lddy, float* dx, int32_t lddx, float* dgamma,
                      float* dbeta, int64_t rows, int32_t C, evk_stream_t stream);
/* LayerNorm(x + dropout_p(res)) with the dropout fused (transformer.py:300-315 `x + dropout(sa)` / `x + dropout(ff)`): the mask
 * is regenerated in the backward from (rng state, sid), which also emits dres = dx * mask / (1-p).  C % 4 == 0, contiguous rows. */
int evk_layernorm_drop_fwd(const float* x, const float* res, const float* gamma, const float* beta, float eps, float p,
                           const uint64_t* rng, uint64_t sid, float* y, float* stats, int64_t rows, int32_t C, evk_stream_t stream);
int evk_layernorm_drop_bwd(const float* x, const float* res, const float* gamma, const float* stats, const float* dy, float p,
                           const uint64_t* rng, uint64_t sid, float* dx, float* dres, float* dgamma, float* dbeta, int64_t rows,
                           int32_t C, evk_stream_t stream);

/* attention softmax (attentions.py:243-279, modules.py:669-682): in place on S [Z][Tq][Tk] (row pitch lds)
 *   s = (S + relk[z][i][j-i+win]) * scale (|j-i|<=win, relk nullable [Z][Tq][2win+1], both unscaled);
 *   key j >= klen[b] or query i >= qlen[b] -> fill (finite -1e4 or -inf); softmax over j.  */
int evk_attn_softmax(float* S, int32_t lds, int32_t Z, int32_t H, int32_t Tq, int32_t Tk, float scale, const float* relk,
                     int32_t win, const int32_t* qlen, const int32_t* klen, float fill, evk_stream_t stream);
/* dS = P * (dP - sum_j dP*P) * scale, in place on dP, and 0 where the forward filled the logit (qlen, klen as given to
 * evk_attn_softmax); also emits drelk[z][i][r] = dS[i][i+r-win] (nullable) */
int evk_attn_softmax_bwd(const float* P, float* dP, int32_t lds, int32_t Z, int32_t H, int32_t Tq, int32_t Tk, float scale,
                         float* drelk, int32_t win, const int32_t* qlen, const int32_t* klen, evk_stream_t stream);
/* Windowed relative-position terms (attentions.py:254-288; skew helpers :312-365 replaced by band indexing).
 * E is [2*win+1][dk] (shared across heads); heads live in the channel dim: q[b][t][h*dk + d].
 *   relk_logits: rel[z][i][r] = q_i . E[r]                        (consumed by evk_attn_softmax)
 *   relk_bwd:    dq_i += sum_r drel[z][i][r] E[r];  dE[r] += sum_{z,i} drel[z][i][r] q_i
 *   attn_band:   band[z][i][r] = P[z][i][i+r-win] (to_band=1) / P[z][i][i+r-win] += band (to_band=0)
 *   relv_out:    out_i += sum_r band[z][i][r] E[r]
 *   relv_bwd:    dband[z][i][r] = dout_i . E[r];  dE[r] += sum_{z,i} band[z][i][r] dout_i            */
int evk_relk_logits(const float* q, int32_t ldq, const float* E, int32_t B, int32_t H, int32_t T, int32_t dk,
                    int32_t win, float* rel, evk_stream_t stream);
int evk_relk_bwd(const float* drel, const float* q, int32_t ldq, const float* E, int32_t B, int32_t H, int32_t T,
                 int32_t dk, int32_t win, float* dq, int32_t lddq, float* dE, evk_stream_t stream);
int evk_attn_band(float* P, int32_t lds, float* band, int32_t Z, int32_t Tq, int32_t Tk, int32_t win, int32_t to_band,
                  evk_stream_t stream);
int evk_relv_out(const float* band, const float* E, int32_t B, int32_t H, int32_t T, int32_t dk, int32_t win,
                 float* out, int32_t ldo, evk_stream_t stream);
int evk_relv_bwd(const float* band, const float* dout, int32_t lddo, const float* E, int32_t B, int32_t H, int32_t T,
                 int32_t dk, int32_t win, float* dband, float* dE, evk_stream_t stream);

/* nearest-codeword search (core_vq.py:172-180): codes[r] = argmax_k -((|x|^2 - 2 x.e_k) + |e_k|^2), lowest
 * index on ties.  The x.E^T products come from evk_sgemm_nt_f32 (exact fp32 FMA, NOT the TF32 tensor path:
 * token indices must not depend on operand rounding).  enorm_scratch: [K] floats. */
int evk_sgemm_nt_f32(const float* A, int32_t lda, const float* B, int32_t ldb, float* C, int32_t ldc, int32_t M,
                     int32_t N, int32_t K, evk_stream_t stream);
int evk_vq_argmax(const float* dots, int32_t ldd, const float* x, int32_t ldx, const float* embed, int32_t lde,
                  int64_t rows, int32_t K, int32_t D, int64_t* codes, float* enorm_scratch, evk_stream_t stream);

/* Trainable quantizer (freeze_quantizer: false; core_vq.py:71-93, 141-149, 203-228, 301-318).  x is [B, T2, D] with row
 * pitch ldx; only rows (b, t < rows_ref[0]) take part (rows_ref: device int32, the reference collate's T / 2).  No float
 * atomics: every sum runs in a fixed order.
 * kmeans_draw: samples = the first n = min(500, B * rows_ref) valid rows in (b, t) order (nsamp[0] = n); means[k] =
 *   samples[idx[k]], idx injected or drawn uniformly from [0, n) with the Philox stream (seed_offset, stream_id); idx_out
 *   (optional) receives the indices.  samples: [500, D], means: [K, D].
 * kmeans_iter: one Lloyd iteration: buckets[i] = argmax_k -sum_d (s_id - m_kd)^2 (direct differences, lowest index on
 *   ties), bins[k] = its count, means[k] = ordered mean of its samples (kept when empty).  buckets: [500] int32.
 * vq_ema: cluster_size <- decay cs + (1 - decay) counts, embed_avg <- decay ea + (1 - decay) (x^T onehot)^T, then
 *   embed <- embed_avg / ((cs + eps) / (sum cs + K eps) * sum cs).  Per code, rows are summed in row order.
 * vq_st_fwd: qst = x + (q - x) [B*T2, D], y = qst upsampled x2 in time [B, 2*T2, D], loss[0] = mean((qst - x)^2) over the
 *   valid rows.  vq_st_bwd: dx = dy[2t] + dy[2t+1] + gloss * 2 (x - qst) / N on valid rows, 0 elsewhere ([B*T2, D]).
 * col_sum: out[c] = sum_r x[r][c] (x dense [rows, C]), chunks of 64 rows added in order. */
int evk_vq_kmeans_draw(const float* x, int32_t ldx, int32_t B, int32_t T2, const int32_t* rows_ref, int32_t K, int32_t D,
                       const int64_t* idx, const uint64_t* seed_offset, uint64_t stream_id, float* samples, int32_t* nsamp,
                       float* means, int64_t* idx_out, evk_stream_t stream);
int evk_vq_kmeans_iter(const float* samples, const int32_t* nsamp, float* means, int32_t K, int32_t D, int32_t* buckets,
                       float* bins, evk_stream_t stream);
int evk_vq_ema(const float* x, int32_t ldx, const int64_t* codes, int32_t B, int32_t T2, const int32_t* rows_ref,
               float* cluster_size, float* embed_avg, float* embed, int32_t K, int32_t D, float decay, float eps,
               evk_stream_t stream);
int evk_vq_st_fwd(const float* x, int32_t ldx, const float* q, int32_t ldq, int32_t B, int32_t T2, int32_t D,
                  const int32_t* rows_ref, float* y, float* qst, float* loss, evk_stream_t stream);
int evk_vq_st_bwd(const float* dy, const float* x, int32_t ldx, const float* qst, int32_t B, int32_t T2, int32_t D,
                  const int32_t* rows_ref, const float* gloss, float* dx, evk_stream_t stream);
int evk_col_sum(const float* x, int64_t rows, int32_t C, float* out, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Loss reductions (losses.py:7-61, sovits.py:513): out[slot] += scale * sum(f(a,b))
 *   kind 0: (1-a)^2   1: a^2   2: |a-b|   ; bwd kinds write da (scaled by *gscale device scalar * scale)
 * ------------------------------------------------------------------------------------------ */
int evk_reduce_loss(int32_t kind, const float* a, const float* b, int64_t n, float scale, float* out,
                    evk_stream_t stream);
int evk_reduce_loss_bwd(int32_t kind, const float* a, const float* b, int64_t n, float scale, const float* gout,
                        float* da, evk_stream_t stream);
/* masked KL (losses.py:46-61): out += sum((logs_p-logs_q-0.5+0.5(z_p-m_p)^2 exp(-2logs_p))*mask); and grads */
int evk_kl_loss(const float* z_p, int32_t ldz, const float* logs_q, int32_t ldq, const float* m_p, int32_t ldm,
                const float* logs_p, int32_t ldp, int32_t B, int32_t T, int32_t C, const int32_t* len, float* out,
                evk_stream_t stream);
int evk_kl_loss_bwd(const float* z_p, int32_t ldz, const float* logs_q, int32_t ldq, const float* m_p, int32_t ldm,
                    const float* logs_p, int32_t ldp, int32_t B, int32_t T, int32_t C, const int32_t* len,
                    const float* gout, float gscale, float* dz_p, float* dlogs_q, float* dm_p, float* dlogs_p,
                    int32_t ldg, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser (sovits.py:286-319,503-525): one fused AdamW pass over a flat fp32 arena (one call per
 * lr group); also accumulates sum(g^2) (commons.py:140-155 grad-norm probe, without its 883 host syncs).
 * ------------------------------------------------------------------------------------------ */
int evk_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n,
                   const float* hyper /* device [lr, step]; bias corrections derived on the device (graph-replay safe) */,
                   float lr_scale, float beta1, float beta2, float eps, float wd, float grad_scale,
                   float* gnorm_sq /* nullable, += */, evk_stream_t stream);
int evk_scalar_add(float* x, float v, evk_stream_t stream);   /* x[0] += v (device-side step counters) */

/* ------------------------------------------------------------------------------------------
 * Dense TF32 GEMM on the TMA-fed persistent wgmma kernel: D[M][N] = epi(A[M][K] * B[N][K]^T + bias[n] + res[m][n]),
 * fp32 storage, row pitches lda/ldb/ldd/ldr in floats (lda, ldb multiples of 4; A, B 16-byte aligned).  This is the
 * kernel evk_gconv_fwd dispatches tap-free (Linear / 1x1 conv) launches to; it is exported for weight gradients on
 * pre-transposed operands: splits > 1 partitions K across CTAs and ACCUMULATES into D, the splits' partials added in split order (D must hold
 * the value to add to, bias/res/act must be null/0).  evk_set_backend_tma(0) routes those launches back to the tap kernel.
 * ------------------------------------------------------------------------------------------ */
int evk_gemm_tf32(const float* A, int32_t lda, const float* B, int32_t ldb, float* D, int32_t ldd, int32_t M, int32_t N,
                  int32_t K, const float* bias, const float* res, int32_t ldr, int32_t act, float slope, int32_t splits,
                  evk_stream_t stream);
int evk_set_backend_tma(int32_t on);
/* Everything a conv's backward needs from its output gradient in one pass (elementwise.cu): g = dy * act'(y) * (t < len*P);
 * dpre (nullable) = g in the layout of dy; dyt (nullable) [B][C][ldt] = g transposed (the K-major operand of evk_gconv_wgrad);
 * dbias (nullable, [C], zero-initialised by the caller) += column sums of g.  act: evk_act of the forward epilogue, yact = its
 * OUTPUT (derivatives are taken from the output: leaky-ReLU / ReLU by sign, tanh by 1 - y^2). */
int evk_dy_prep(const float* dy, int32_t lddy, const float* yact, int32_t ldy, int32_t act, float slope, float gscale, const int32_t* len,
                int32_t P, float* dpre, int32_t ldp, float* dyt, int32_t ldt, int64_t t_sb, float* dbias, int32_t B, int32_t T, int32_t C,
                evk_stream_t stream);
/* gscale multiplies g: 1/(1-p) when the forward epilogue applied dropout after a ReLU -- the saved OUTPUT is then zero exactly
 * where the element was dropped or the ReLU was off, so no mask needs to be regenerated. */
/* [B][T][ldx] (C valid, batch pitch x_sb) -> [B][C][ldy] (T + shift valid, batch pitch y_sb):
 * y[b][c][u] = x[b][u - shift][c], zero for u < shift. */
int evk_transpose_rows(const float* x, int32_t ldx, int64_t x_sb, float* y, int32_t ldy, int64_t y_sb, int32_t B, int32_t T,
                       int32_t C, int32_t shift, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage-1 AR semantic-token GPT (t2s_model.py:431-490 forward_old, transformer.py:266-315, optim.py:123-622).
 * Linear layers / LayerNorm / embedding / dropout reuse the entry points above.
 * ------------------------------------------------------------------------------------------ */
/* Fused prefix-LM attention, head dim 32.  q/k/v: [B, L, ld] with head h at columns h*32.. (three column blocks of the
 * in_proj output).  Key j is visible to query i iff (j < X ? j < xlen[b] : (j - X < ylen[b] && j <= i)), which is the
 * mask built at t2s_model.py:456-479; scores and mask are never materialised.  lse: [B*H, L] (log2 domain) is saved for
 * the backward.  p_drop applies to the probabilities as F.scaled_dot_product_attention(dropout_p) does; the keep mask is
 * a counter hash of (rng[0]=seed, rng[1]=offset, sid, b, h, i, j), regenerated in the backward. */
int evk_flash_attn_fwd(const float* q, const float* k, const float* v, int32_t ld, float* o, int32_t ldo, float* lse, int32_t B,
                       int32_t H, int32_t L, int32_t X, int32_t dk, const int64_t* xlen, const int64_t* ylen, float scale,
                       float p_drop, const uint64_t* rng, uint64_t sid, evk_stream_t stream);
/* delta: [B*H, L] scratch (written).  dq/dk/dv: [B, L, lddq] (+ h*32), every element written. */
int evk_flash_attn_bwd(const float* q, const float* k, const float* v, int32_t ld, const float* o, int32_t ldo,
                       const float* lse, const float* dout, int32_t lddo, float* delta, float* dq, float* dk, float* dv,
                       int32_t lddq, int32_t B, int32_t H, int32_t L, int32_t X, int32_t dkdim, const int64_t* xlen,
                       const int64_t* ylen, float scale, float p_drop, const uint64_t* rng, uint64_t sid, evk_stream_t stream);
/* SinePositionalEmbedding with learnable alpha (embedding.py:36-81): y[b][t] = x[b][t] + alpha[0] * pe[t]; *_sb are batch
 * strides in floats so y can be a row range of the concatenated [B, X+Y, D] sequence.  bwd: dalpha[0] += <dy, pe>. */
int evk_sinepos_add(const float* x, int32_t ldx, int64_t x_sb, const float* pe, int32_t ldpe, const float* alpha, float* y,
                    int32_t ldy, int64_t y_sb, int32_t B, int32_t T, int32_t D, evk_stream_t stream);
int evk_sinepos_bwd(const float* dy, int32_t ldy, int64_t dy_sb, const float* pe, int32_t ldpe, float* dalpha, int32_t B,
                    int32_t T, int32_t D, evk_stream_t stream);
/* CrossEntropyLoss(reduction="sum") + MulticlassAccuracy(top_k, micro, ignore_index) (t2s_model.py:486-489).
 * out2[0] = sum_r (lse_r - logit_r[target_r]); out2[1] = #hits / #valid, hit = fewer than top_k logits strictly above
 * the target's.  lse/nll: [rows] scratch kept for the backward; flags: [rows] bytes.
 * bwd: dl[r][c] = gscale[r / rows_per_g] * (softmax(logits_r)[c] - [c == target_r]). */
/* Skinny Linear of the KV-cache token step (decode_next_token, t2s_model.py:187-221: one new row per utterance):
 * y[r][n] = act(sum_c x[r][c] * W[n][c] + bias[n]) for rows <= 64; W = the packed forward operand PA[0] ([N][ldw], row n = output
 * channel n).  Exact fp32 FMAs, one pass over W.  A row's result does not depend on `rows` (same summation order for every
 * batch size).  rows <= 4 requires rows_rounded_up_to_a_power_of_2 * C * 4 bytes <= 40 KB (gemv_rows_fit in csrc/gemv_route.h).
 * act: EVK_ACT_NONE / RELU / LRELU. */
int evk_gemv_rows(const float* x, int32_t ldx, int32_t rows, const float* W, int32_t ldw, const float* bias, float* y,
                  int32_t ldy, int32_t N, int32_t C, int32_t act, float slope, evk_stream_t stream);
/* 16-bit Linears (csrc/linear_h16.cu; Whisper's float16 / bfloat16 compute types).  Numerical contract:
 *   y[r][n] = act( sum_k h(x[r][k]) * h(W[n][k]) + bias[n] + res[r][n] )
 * h = round to nearest even to fp16 (bf16 == 0) or bf16 (bf16 != 0): applied to the fp32 activations as they are staged
 * (cvt.rn; values beyond fp16's range become +-inf as that cast makes them) and to the weight once, when it is packed.
 * The products are formed on tensor cores and accumulated in fp32; a product of two fp16 or two bf16 values is exact in
 * fp32, so only the accumulation rounds.  The epilogue (bias, res, act) is fp32, in that order.  evk_set_precise has no
 * effect here: the operands are already exact.  Each output has one K order whatever `rows` is, so a row's bits never depend
 * on its neighbours or on how many rows share the launch.
 * W: the packed weight [N][ldw] 16-bit (fp16 or bf16 bits as selected), ldw % 64 == 0, ldw >= K, columns K .. ldw - 1 zero,
 * 16-byte aligned (ops.pack_weight_h16).  x [rows][ldx] fp32, ldx >= K (columns past K are never read); y [rows][ldy];
 * res [rows][ldr] or null; bias [N] or null; act: any evk_act (slope for LRELU).  Both entry points take the same operands.
 *   evk_linear_rows_h16: the few rows of a decode step, any row count (mma.sync.m16n8k16).  Each CTA streams its slice of W
 *     once per 128 rows; the K range is split over CTAs by (N, K) alone, and the splits' fp32 partials are added in split
 *     order (library scratch).
 *   evk_linear_h16: many rows (wgmma.m64n128k16 from TMA-loaded shared memory): x is first cast to 16 bits in library
 *     scratch ([rows][K rounded up to 8]).  No K split.  rows <= 65535 * 128.
 * The two entry points may differ from each other in the last bits of a sum (their K orders differ). */
int evk_linear_rows_h16(const float* x, int32_t ldx, int32_t rows, const void* w, int32_t ldw, int32_t bf16, const float* bias,
                        const float* res, int32_t ldr, float* y, int32_t ldy, int32_t N, int32_t K, int32_t act, float slope,
                        evk_stream_t stream);
int evk_linear_h16(const float* x, int32_t ldx, int32_t rows, const void* w, int32_t ldw, int32_t bf16, const float* bias,
                   const float* res, int32_t ldr, float* y, int32_t ldy, int32_t N, int32_t K, int32_t act, float slope,
                   evk_stream_t stream);
/* KV-cache attention of one new token -- T2SBlock.decode_next_token (t2s_model.py:203-221), F.scaled_dot_product_attention
 * without mask -- with the position in DEVICE memory, so that a decode step replays as a CUDA graph.  qkv: the in_proj outputs
 * [q | k | v] (3 * H * 32 floats per row, pitch ld, batch stride `batch_stride`) of the positions so far; *n_prev_dev = rows
 * already in the cache before this token.  evk_cache_append writes the token's row at that index; evk_attn_decode_dev attends
 * rows 0 .. *n_prev_dev with the q block of row *n_prev_dev as the query.  out [B, H * 32] (pitch ldo).  Exact fp32.
 * skip: NULL, or device [B][2]: item b leaves out keys skip[b][0] .. skip[b][1] - 1 (the right padding of its text when a batch
 * is padded to a common text length: skip[b] = (x_len_b, max_len)). */
int evk_attn_decode_dev(const float* qkv, int64_t batch_stride, int32_t ld, const int32_t* n_prev_dev, const int32_t* skip,
                        int32_t B, int32_t H, float scale, float* out, int32_t ldo, evk_stream_t stream);
int evk_cache_append(const float* row, int32_t ldr, float* cache, int64_t batch_stride, int32_t ld, const int32_t* pos_dev,
                     int32_t B, int32_t W, evk_stream_t stream);
/* The same token step on a 16-bit K/V cache (the stage-1 GPT's float16 / bfloat16 compute type), one launch per layer in
 * place of evk_cache_append + evk_attn_decode_dev.  cache: [B][rows][2 * H * 32] 16-bit values, k then v (no q columns), row
 * pitch ld elements and batch stride batch_stride elements, both multiples of 8, 16-byte aligned; bf16 != 0 selects bf16,
 * else fp16.  row: this step's in_proj output [B][3 * H * 32] fp32 ([q | k | v]), pitch ldr (a multiple of 4, 16-byte
 * aligned).  The CTA of (head h, item b) stores h(k) and h(v) of head h at cache row *n_prev_dev (h = round to nearest even,
 * cvt.rn; it writes only its own head's 64 values) and attends keys 0 .. *n_prev_dev -- the current key with its rounded k
 * and v -- with the fp32 q block of `row` times `scale` as the query.  Numerical contract: the 16-bit k and v are widened
 * exactly; scores, the online softmax, its sums and P V are fp32, in evk_attn_decode_dev's order (thread t owns the same keys
 * whatever B and the padding are), so an item's bits do not depend on the other items of the launch.  skip as for
 * evk_attn_decode_dev: keys skip[b][0] .. skip[b][1] - 1, and rows past *n_prev_dev, are never read.  out [B][ldo] fp32. */
int evk_attn_decode_h16(const float* row, int32_t ldr, void* cache, int64_t batch_stride, int32_t ld, int32_t bf16,
                        const int32_t* n_prev_dev, const int32_t* skip, int32_t B, int32_t H, float scale, float* out, int32_t ldo,
                        evk_stream_t stream);
/* Fused token sampler of batched KV-cache decoding (infer_panel_batch_infer, t2s_model.py:563-730; utils.py:109-157), one CTA
 * per row b of logits [B][ldl] (V <= 2048 classes, eos = V - 1), in the reference's order: repetition penalty over the row's
 * history (prompt included) -> top-p if top_p < 1 (descending order, cumulative softmax, `cum > top_p` removed, the first kept;
 * on the penalised, un-tempered logits) -> / max(T, 1e-5) -> top-k (values >= the k-th largest kept) -> softmax ->
 * argmax(p / q), q ~ Exp(1).  The step is idx = *n_dev - icfg[2]; at idx < eos_steps (>= 0) EOS is excluded (the batched
 * decoders pass 1; infer_panel_naive, t2s_model.py:835-836, passes 11, with a prompt or without one).  The row stops when
 * the token or the argmax of the penalised logits is EOS (fin[b] = (idx, idx - 1)), else when idx + 1 > early_stop (!= -1)
 * or idx == max_steps - 1 (fin[b] = (idx, idx)); a row with fin[b][0] >= 0 is left untouched.  Otherwise hist[b][prefix +
 * idx] = token, its bit is set in seen, and x_next[b] = emb[token] + alpha[0] * pe[prefix + idx].
 *   icfg: device int64 [6] = (seed, prefix, n0, top_k >= 1, early_stop, max_steps);  fcfg: device float [3] = (top_p, T, penalty)
 *   q: NULL (counter-based Exp(1) draws keyed by (seed, row, idx, class)) or supplied draws [B][ldq]
 *   hist: int64 [B][ldh];  seen: uint32 [B][(V + 31) / 32] bitmap of the tokens in hist;  fin: int32 [B][2], -1 while running
 *   emb: [V][D], pe: [*][D], x_next: [B][D]. */
int evk_sample_tokens(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, int32_t eos_steps,
                      const int64_t* icfg, const float* fcfg, const int32_t* n_dev, const float* q, int32_t ldq, int64_t* hist,
                      int32_t ldh, uint32_t* seen, int32_t* fin, const float* emb, const float* pe, const float* alpha,
                      float* x_next, int32_t D, evk_stream_t stream);
/* evk_sample_tokens with one configuration per row (tts.run_many decodes rows of several requests together), no supplied
 * draws:  icfg: device int64 [B][8], row b = (seed, prefix, n0, top_k >= 1, early_stop, max_steps, eos_steps >= 0, key row);
 * fcfg: device float [B][4], row b = (top_p, T, penalty, unused).  Row b's Exp(1) draws are keyed by (its seed, its key row,
 * idx, class) instead of (seed, b, idx, class), so a row samples what it would sample at row `key row` of a batch decoded with
 * evk_sample_tokens and that seed, whichever rows share the launch. */
int evk_sample_tokens_rows(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, const int64_t* icfg,
                           const float* fcfg, const int32_t* n_dev, int64_t* hist, int32_t ldh, uint32_t* seen, int32_t* fin,
                           const float* emb, const float* pe, const float* alpha, float* x_next, int32_t D, evk_stream_t stream);
/* Cross entropy over rows [B][T] of positions (row r is position r % T).  count: NULL (every row counts; T is then unused), or
 * a device int32 scalar n: positions t >= n add no loss, no accuracy count (neither valid nor hit) and no gradient (evk_ce_bwd
 * writes 0 to their logit gradients).  The bound is for batches padded past the collate's length (the stage-1 trainer pads to
 * a 32-token grid so that a CUDA graph can serve many batches): the reference sums CE over every position of its padded batch
 * (EOS targets included), so positions added by further padding must not count. */
int evk_ce_fwd(const float* logits, int32_t ld, const int64_t* targets, int32_t rows, int32_t V, int32_t topk,
               int64_t ignore_index, const int32_t* count, int32_t T, float* lse, float* nll, uint8_t* flags, float* out2,
               evk_stream_t stream);
int evk_ce_bwd(const float* logits, int32_t ld, const int64_t* targets, const float* lse, const float* gscale,
               int32_t rows_per_g /* row r is scaled by gscale[r / rows_per_g]; == rows for one scalar */, const int32_t* count,
               int32_t T, float* dl, int32_t lddl, int32_t rows, int32_t V, evk_stream_t stream);
/* DPO head of Text2SemanticDecoder.forward (t2s_model.py:393-429; utils.py:160-192 with reference_free=True): from the
 * per-token nll of the chosen [B, Yc] and rejected [B, Yr] sequences: out3 = (sum CE of chosen, mean_b -logsigmoid(beta *
 * (logp_chosen_b - logp_rejected_b)), their sum); coef_c/coef_r [B] = d out3[2] / d nll_{c,r}[b][t] (feeds evk_ce_bwd).
 * count_c / count_r: NULL, or device int32 scalars; the per-row log-prob sums (and so loss_1) then run over
 * t < min(Yc, *count_c) resp. t < min(Yr, *count_r).  The stage-1 trainer passes the collate's Y for the chosen branch and
 * max(reject_lens) for the rejected one. */
int evk_dpo_head(const float* nll_c, int32_t Yc, const int32_t* count_c, const float* nll_r, int32_t Yr,
                 const int32_t* count_r, int32_t B, float beta, float* out3, float* coef_c, float* coef_r, evk_stream_t stream);
/* Rejected rows of the DPO variant (utils.py:195-232, the repeat branch) from host-drawn spans, capturable in a CUDA graph:
 * row b of y [B][ldy] (int64, padded chosen rows) with span (i0, i1) = spans[b] (int32 [B][2], 0 <= i0 <= i1 <= Yc) becomes
 *   out[b] = y[b][:i0] ++ y[b][i0:i1] ++ y[b][i0:i1] ++ y[b][i1:Yc]  followed by 0 up to Yr   (out: int64 [B][Yr])
 * and lens[b] = Yc + i1 - i0 (int64).  yc: device int32 scalar Yc (<= ldy), the collate's width of y.  Every row must fit:
 * Yc + i1 - i0 <= Yr (positions past Yr are not written). */
int evk_dpo_reject_rows(const int64_t* y, int32_t ldy, int32_t B, const int32_t* spans, const int32_t* yc, int64_t* out,
                        int32_t Yr, int64_t* lens, evk_stream_t stream);
/* ScaledAdam (optim.py:123-622) over flat arenas p/g/delta/v.  chunks: [nchunks][3] = (tensor id, begin, count), numel: [nt].
 * Per-tensor state: rms, sv (scale_exp_avg_sq) [nt]; sg (scale_grads) [size_update_period][nt]; stats [nt][3] and
 * coef [nt][2] are scratch (stats must be zero on first use; the call leaves it zero).  hyper: device [lr];
 * stepbuf: device step counter (incremented); norms: [clipping_update_period]; thr: [2] = (threshold, valid);
 * glob: [4] scratch (glob[2] = clipping scale of this step).  Gradients are read as g * gscale; zero_grad != 0 clears g.
 * Three launches (per-tensor reductions, per-tensor scalars + median clipping, fused update); no host sync. */
int evk_scaled_adam(float* p, float* g, float* delta, float* v, const int64_t* chunks, int32_t nchunks, const int64_t* numel,
                    int32_t nt, float* stats, float* rms, float* sv, float* sg, float* coef, const float* hyper,
                    int64_t* stepbuf, float* norms, float* thr, float* glob, float gscale, float beta1, float beta2,
                    float clipping_scale, int32_t clipping_update_period, float scalar_lr_scale, float eps,
                    float param_min_rms, float param_max_rms, float scalar_max, int32_t size_update_period,
                    int32_t zero_grad, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * BERT text features (Normalize._get_bert_feature, normalize.py:88-106; TextPreprocessor.get_bert_feature,
 * inference/preprocessor.py:180-193).  Linear layers / LayerNorm / GELU / embedding reuse the entry points above.
 * ------------------------------------------------------------------------------------------ */
/* Fused bidirectional attention with per-row key lengths, head dim 64, inference only:
 *   O = softmax(Q K^T * scale + mask) V   per (batch b, head h),   mask: key j is visible to every query iff j < lens[b].
 * q/k/v: [B, L, ld] with head h at columns h*64.. (usually the three column blocks of one packed QKV Linear output);
 * o: [B, L, ldo].  Requires 1 <= lens[b] <= L (lens: int64 device [B], values outside are clamped to [1, L]),
 * ld % 4 == 0, ldo % 2 == 0, q/k/v 16-byte and o 8-byte aligned.  L has no upper bound: keys stream through in tiles of 32
 * and only the tiles that hold a visible key are read (BERT's 512-position limit is enforced by its caller).  Query rows at
 * or past lens[b] are computed like any other (finite).  Scores are never materialised (online softmax); TF32 mma.sync with fp32 accumulation (3xTF32 under
 * evk_set_precise(1)); no atomics, bit-reproducible. */
int evk_attn_pad_fwd(const float* q, const float* k, const float* v, int32_t ld, float* o, int32_t ldo, int32_t B,
                     int32_t H, int32_t L, const int64_t* lens, float scale, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * UVR5 VR separation (CascadedASPPNet and the DeEcho / DeReverb CascadedNet, uvr5.py), inference only.  Activations are
 * channels-last fp32: pixel (b, y, x) of an operand starts at  p + b*bs + (y*W + x)*pitch  (floats), so a channel slice of
 * a concat buffer is an operand.
 * ------------------------------------------------------------------------------------------ */
enum evk_conv2d_act { EVK_C2_NONE = 0, EVK_C2_RELU = 1, EVK_C2_LRELU = 2 /* slope 0.01 */, EVK_C2_SIGMOID = 3,
                      EVK_C2_GELU = 4 /* exact erf */ };
/* y = act(conv2d(x, w) * scale[n] + bias[n])  (scale / bias may be null: 1 / 0).  x: [B, H, W, C] (pitch x_pitch >= C,
 * batch stride x_bs); w: [N][k][k][C] (k = 1, 2 or 3); stride 1 or 2, zero padding and dilation >= 1 per axis (the DeEcho /
 * DeReverb ASPP: dilation (4, 2), (8, 4), (12, 6)); y: [B, Ho, Wo, N] (pitch y_pitch >= N, batch stride y_bs),
 * Ho = (H + 2 pad_h - dil_h (k - 1) - 1) / stride + 1, Wo likewise with pad_w, dil_w.  Implicit GEMM with TF32
 * products and fp32 accumulation: wgmma when C, x_pitch and x_bs are multiples of 4 and x, w are 16-byte aligned,
 * mma.sync otherwise and for 3xTF32 under evk_set_precise(1).  No atomics, and every output's sum has one order whatever
 * B is, so results are bit-reproducible and independent of the batch. */
int evk_conv2d_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, const float* scale, const float* bias,
                   float* y, int32_t y_pitch, int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t N, int32_t k,
                   int32_t stride, int32_t pad_h, int32_t pad_w, int32_t dil_h, int32_t dil_w, int32_t act,
                   evk_stream_t stream);
/* evk_conv2d_fwd with 16-bit products (the VR, DeEcho / DeReverb and MDX23C float16 / bfloat16 compute types): the same
 * operands, geometry and epilogue, and a packed 16-bit weight.  Numerical contract:
 *   acc[m][n] = sum_k h(x[m][k]) * h(w[n][k])   over K = k*k*C in evk_conv2d_fwd's order (tap-major, channel-minor),
 *   y = act(acc * scale[n] + bias[n])
 * h = round to nearest even to fp16 (bf16 == 0) or bf16 (bf16 != 0): applied to the fp32 activations as they are staged
 * (cvt.rn; values beyond fp16's range become +-inf as that cast makes them) and to the weight once, when it is packed.  A
 * product of two 16-bit values is exact in fp32 and the accumulation is fp32; scale and bias stay in the fp32 epilogue
 * (BatchNorm's scale is not folded into the 16-bit weight, so a weight from an fp16 checkpoint keeps its bits).  No atomics
 * and no K split: every output is summed in one K order (slabs of 64 in K order) whatever B is, so a window's bits are the
 * same alone or batched.  evk_set_precise has no effect here.  Any C, pitch and channel offset is read in place (16-, 8- or
 * 4-byte loads as alignment allows); input channels outside [0, C) of a pixel are never read.
 * w: [N][ldw] fp16 or bf16 bits, row n = w[n][ky][kx][c] in K order, ldw % 64 == 0, ldw >= k*k*C, columns past k*k*C zero,
 * 16-byte aligned (ops.pack_conv_h16).  wgmma.m64nNk16 on tiles of 128 output pixels by 16 / 32 / 64 / 128 channels (the
 * smallest that covers N, 128 for wider layers). */
int evk_conv2d_fwd_h16(const float* x, int32_t x_pitch, int64_t x_bs, const void* w, int32_t ldw, int32_t bf16,
                       const float* scale, const float* bias, float* y, int32_t y_pitch, int64_t y_bs, int32_t B, int32_t H,
                       int32_t W, int32_t C, int32_t N, int32_t k, int32_t stride, int32_t pad_h, int32_t pad_w, int32_t dil_h,
                       int32_t dil_w, int32_t act, evk_stream_t stream);
/* Depthwise 3x3, stride 1, zero padding = dil: y[b,y,x,c] = sum_{i,j} w[c][i][j] x[b, y + (i-1) dil, x + (j-1) dil, c]
 * (fp32 FMA).  w: [C][3][3]. */
int evk_dwconv3x3_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, float* y, int32_t y_pitch,
                      int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t dil, evk_stream_t stream);
/* Bilinear resize [B, Hi, Wi, C] -> [B, Ho, Wo, C] with align_corners=True (F.interpolate's index and weight rules; an
 * input extent of 1 broadcasts). */
int evk_resize_bilinear_ac(const float* x, int32_t x_pitch, int64_t x_bs, int32_t Hi, int32_t Wi, float* y,
                           int32_t y_pitch, int64_t y_bs, int32_t Ho, int32_t Wo, int32_t B, int32_t C,
                           evk_stream_t stream);
/* y[b][x][c] = mean_y x[b, y, x, c]  (AdaptiveAvgPool2d((1, None))); y: contiguous [B, 1, W, C]. */
int evk_mean_h(const float* x, int32_t x_pitch, int64_t x_bs, float* y, int32_t B, int32_t H, int32_t W, int32_t C,
               evk_stream_t stream);
/* Mask head of CascadedASPPNet.predict (nets.py:60-122): h [B, max_bin, W, Ch] (pitch / batch stride), w [2][Ch] (the
 * bias-free 1x1 output conv), mix NCHW [B, 2, out_bin, W] ->
 *   out[b, c, r, x - offset] = mask(c, min(r, max_bin - 1), x)^e(r) * mix[b, c, r, x]   for offset <= x < W - offset,
 * mask = sigmoid(w[c] . h), e(r) = e_lo for r < split_bin, e_hi otherwise, and 1 when use_agg == 0.
 * out: contiguous [B, 2, out_bin, W - 2 offset]. */
int evk_vr_mask_head(const float* h, int32_t h_pitch, int64_t h_bs, const float* w, int32_t Ch, const float* mix,
                     float* out, int32_t B, int32_t max_bin, int32_t out_bin, int32_t W, int32_t offset, int32_t split_bin,
                     float e_lo, float e_hi, int32_t use_agg, evk_stream_t stream);
/* Recurrence of a bidirectional one-layer nn.LSTM (gate order i, f, g, o; zero initial h and c), inference only.
 * g: the input projections with both biases added, row (t, n) at g + t*g_st + n*g_sn holding 8H floats
 * [direction][gate][H] (direction 0 forward, 1 reverse); w_hh: [2][4H][H] (weight_hh_l0, weight_hh_l0_reverse);
 * y: row (t, n) at y + t*y_st + n*y_sn receives [h_forward(t) | h_reverse(t)] (2H floats).  Strides are in floats, so
 * (t, n) and (n, t) row orders both work.  H = 32 or 64 (EVK_ERR_ARG otherwise).  One persistent launch, W_hh held
 * on chip; exact fp32 FMAs, accurate expf / tanhf, no atomics: bit-reproducible, and a row's result does not depend on
 * the other rows of the batch. */
int evk_lstm_bidir_fwd(const float* g, int64_t g_st, int64_t g_sn, const float* w_hh, float* y, int64_t y_st, int64_t y_sn,
                       int32_t T, int32_t N, int32_t H, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * UVR5 BS-Roformer separation (BSRoformer, bs_roformer.py), inference only.  Linear layers run on evk_gconv_fwd, the mask
 * estimator's GLU on evk_glu_res, the forward STFT on evk_stft_fwd.
 * ------------------------------------------------------------------------------------------ */
/* Fused axial self-attention with rotary embedding and per-head gates, head dim 64, no mask (Attention.forward of
 * bs_roformer.py:106-121 from the QKV output to just before to_out).  A token row of qkvg (pitch ld floats) is
 * [q (H*64) | k (H*64) | v (H*64) | gate logits (H)] (to_qkv and to_gates as one Linear).  q and k are rotated at their
 * position p = 0 .. L-1 in the sequence with interleaved pairs, out[2i] = x[2i] cos - x[2i+1] sin and out[2i+1] =
 * x[2i+1] cos + x[2i] sin, where cs [L][32][2] holds (cos, sin) of the angle p * theta_i; then
 *   o = softmax(q k^T / 8) v * sigmoid(gate_h),  written as [h*64 + d] of the token's row of o (pitch ldo).
 * Sequences: n = (u, w), u < n_outer, w < n_inner; token t of sequence n is row u*s_outer + w*s_inner + t*s_tok of both
 * qkvg and o (strides in rows).  [B, T, F, C] activations: time axis n_outer = B, s_outer = T*F, n_inner = F, s_inner = 1,
 * s_tok = F; frequency axis n_outer = B*T, s_outer = F, n_inner = 1, s_inner = 0, s_tok = 1.  Any L >= 1 (online softmax
 * over 32-key tiles).  ld % 4 == 0, ldo % 2 == 0; qkvg 16-byte, o and cs 8-byte aligned.  TF32 mma.sync with fp32
 * accumulation (3xTF32 under evk_set_precise(1)); no atomics, bit-reproducible. */
int evk_rope_attn_fwd(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                      int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok, evk_stream_t stream);
/* The same attention with 16-bit operands (the Roformers' float16 / bfloat16 compute types): the operands, geometry and
 * strides of evk_rope_attn_fwd, and h = round to nearest even to fp16 (bf16 == 0) or bf16 (bf16 != 0).  Numerical contract:
 *   q and k are rotated in fp32 with the cs table and the formula above, then rounded with h; v is rounded with h.
 *   s = h(q_rot) . h(k_rot) on mma.sync.m16n8k16 (products exact, fp32 accumulation), times 1/8.
 *   The online softmax is fp32 and the same as evk_rope_attn_fwd's (running maxima and sums over 32-key tiles, ex2.approx);
 *   its sums add the fp32 probabilities p.
 *   o = (sum_j h(p_j) h(v_j)) / (sum_j p_j) * sigmoid(gate), P . V accumulated in fp32, the gate in fp32.
 * Values beyond fp16's range become +-inf under h.  No atomics: a sequence's output depends only on that sequence, so it is
 * bit-identical whatever n_outer / n_inner are.  evk_set_precise has no effect here. */
int evk_rope_attn_fwd_h16(const float* qkvg, int32_t ld, const float* cs, float* o, int32_t ldo, int32_t H, int32_t L,
                          int32_t n_outer, int64_t s_outer, int32_t n_inner, int64_t s_inner, int64_t s_tok, int32_t bf16,
                          evk_stream_t stream);
/* Inverse of evk_stft_fwd's center=True transform with the periodic Hann(n_fft) window: torch.istft(n_fft, hop, n_fft, hann,
 * center=True, normalized=False, onesided=True, length=length or None) of cplx [B*S*T][n_fft/2+1][2] (rows b*S + s), times
 * mask when given (bs_roformer.py:530-543): bin k of row (b, s), frame t is multiplied by the complex mask at columns
 * 2 (k S + s) .. +1 of mask row b*T + t (pitch ld_mask: the mask estimator's 'b t (f s c)' layout).  Per frame a C2R inverse
 * DFT (imaginary parts of bins 0 and n_fft/2 ignored) and the window, written to work [B*S*T][n_fft]; then the overlap-add in
 * frame order, divided by the sum of squared windows, trimmed by n_fft/2 at both ends: out [B*S][ld_out] gets hop*(T-1)
 * samples per row when length == 0, else torch.istft's length=length: `length` samples per row, computed by the same
 * overlap-add (past hop*(T-1) from the frames' tails), 0 < length < hop*(T-1) + n_fft/2; a negative length is EVK_ERR_ARG.
 * n_fft a power of two in [256, 8192], or an even divisor of 61440 (2^12 3 5) in [16, 7680] (the mixed-radix core: the
 * UVR5 VR band sizes 320, 640, 960); T >= 2, hop <= n_fft / 2, B*S <= 65535. */
int evk_istft(const float* cplx, const float* mask, int32_t ld_mask, int32_t B, int32_t S, int32_t T, int32_t n_fft, int32_t hop,
              int32_t length, float* work, float* out, int32_t ld_out, evk_stream_t stream);
/* Band-split operand (bs_roformer.py:481-490, mel_band_roformer.py:419-425, and each band's RMSNorm before its Linear):
 * from evk_stft_fwd's cplx [B*S*T][n_bins][2] (rows b*S + s) to y [B*T][ld_y], row (b, t), column (j S + s) * 2 + c for
 * slot j of the bin table (bin bins[j]; 'b t (f s c)'), with the columns [2 S band_off[i], 2 S band_off[i+1]) of band i
 * divided by max(their L2 norm, 1e-12).  band_off: device int32 [n_bands + 1]; bins: device int32 [band_off[n_bands]], each
 * < n_bins (BS-Roformer: the identity table 0 .. n_bins-1).  S = 1 or 2; 2 S n_bins floats must fit 48 KB;
 * ld_y >= 2 S band_off[n_bands]. */
int evk_band_input(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, const int32_t* band_off,
                   const int32_t* bins, int32_t n_bands, float* y, int32_t ldy, evk_stream_t stream);
/* y[r] = x[r] / max(||x[r]||_2, 1e-12) per row when gamma == NULL (F.normalize(dim=-1): the RMSNorms whose gamma * sqrt(dim)
 * the caller folds into the next Linear's weight columns), else that times sqrt(C) * gamma (RMSNorm with its gamma, the
 * output norm of each Mel-Band Roformer Transformer; in fp32 in that order; gamma: device [C]).  y may be x (in place,
 * ldy == ldx). */
int evk_row_norm(const float* x, int32_t ldx, const float* gamma, float* y, int32_t ldy, int64_t rows, int32_t C,
                 evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * UVR5 MDX23C (the TFC-TDF v3 U-Net, mdx23c.py; lib_v5/vr_network/tfc_tdf_v3.py), mdx23c.cu, inference only.  Activations are
 * channels-last fp32 [B, H, W, C] with the spatial axes (time frames, frequency bins), as the VR nets' operands above.  The
 * 3x3, 1x1 and 2x2 stride-2 convolutions run on evk_conv2d_fwd, the instance norms on evk_instnorm_plane.
 * ------------------------------------------------------------------------------------------ */
/* TDF Linear along the frequency axis: for every slab z < Z (one (item, frame) row of W = K pixels),
 *   y[z][m][n] = sum_k a[m][k] x[z][k][n] (+ r[z][m][n])
 * a: the Linear's weight [M][K] contiguous; x row k of slab z at x + z x_zs + k ldx (ldx = the pixel pitch), likewise r, y.
 * r may be y (in place).  TF32 mma.sync with fp32 accumulation in one K order (3xTF32 under evk_set_precise(1)); no atomics,
 * bit-reproducible and independent of Z. */
int evk_mdx_tdf(const float* a, const float* x, int32_t ldx, int64_t x_zs, const float* r, int32_t ldr, int64_t r_zs,
                float* y, int32_t ldy, int64_t y_zs, int32_t Z, int32_t M, int32_t N, int32_t K, evk_stream_t stream);
/* ConvTranspose2d(C, N, kernel 2, stride 2, no bias): y[b, 2i + dy, 2j + dx, n] = sum_c x[b, i, j, c] w[dy][dx][n][c]
 * (w: the reference's [C][N][2][2] weight as [2][2][N][C]).  x [B, H, W, C] (pitch x_pitch, x_bs = H W x_pitch), y [B, 2H,
 * 2W, N] (pitch y_pitch, y_bs = 4 H W y_pitch): a channel slice of a concat buffer.  Four evk_conv2d_fwd 1x1 launches, one
 * per output phase, with its precision, determinism and batch independence. */
int evk_convt2x2_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, float* y, int32_t y_pitch, int64_t y_bs,
                     int32_t B, int32_t H, int32_t W, int32_t C, int32_t N, evk_stream_t stream);
/* STFT -> U-Net input (STFT.__call__ and cac2cws): from evk_stft_fwd's cplx [B*S*T][n_bins][2] (rows b*S + s) to
 * y[b, t, j, (2 s + c) k + u] = cplx[b S + s][t][u F + j][c], j < F, u < k: the first k F bins, channels (s, re/im, subband),
 * pixel (t, j) at y + ((b T + t) F + j) ldy. */
int evk_mdx_front(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, int32_t k, int32_t F, float* y,
                  int32_t ldy, evk_stream_t stream);
/* final_conv output -> evk_istft's input (cws2cac, the target split and STFT.inverse's zero bins): x [B, T, F, ldx] holding
 * nt * 2 S k channels to cplx [(b nt + g) S + s][t][f][c] = x[b, t, f % F, g 2 S k + (2 s + c) k + f / F] for f < k F, 0 up
 * to n_bins. */
int evk_mdx_back(const float* x, int32_t ldx, int32_t B, int32_t nt, int32_t S, int32_t T, int32_t n_bins, int32_t k, int32_t F,
                 float* cplx, evk_stream_t stream);
/* y[p][c] = (a[p][c] + b[p][c]) * m[p][c] for P pixels of C channels (row pitches lda, ldb, ldm, ldy; m nullable: no product):
 * the TFC-TDF residual adds, and the last one's `x * first_conv_out`. */
int evk_mdx_add(const float* a, int32_t lda, const float* b, int32_t ldb, const float* m, int32_t ldm, float* y, int32_t ldy,
                int64_t P, int32_t C, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Mel-Band Roformer (mel_band_roformer.py; lib_v5/vr_network/mel_band_roformer.py:244-478), roformer.cu.  The bands
 * overlap: band i holds the bins bins[band_off[i] .. band_off[i+1]) (ascending), and a bin may belong to two bands.
 * ------------------------------------------------------------------------------------------ */
/* Averaged mask (mel_band_roformer.py:455-466): g [rows][ldg] holds the mask estimators' complex outputs in the band-split
 * column order of evk_band_input.  mask [rows][ld_mask] at columns 2 (f S + s) .. +1 (evk_istft's mask layout) gets the
 * sum over k in [cover_off[f], cover_off[f+1]) of g's complex pair (cover[k] S + s), summed in that order, divided by the
 * count cover_off[f+1] - cover_off[f] (>= 1).  cover lists the slots of bin f in ascending band order.  No atomics. */
int evk_melband_mask_avg(const float* g, int32_t ldg, const int32_t* cover_off, const int32_t* cover, int32_t S, int32_t n_bins,
                         int64_t rows, float* mask, int32_t ld_mask, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * UVR5 VR front and back end (SeparateVR.separate, uvr5/separate.py:103-196; spec_utils.py), vr_wave.cu.  Frame sizes are
 * those of the mixed-radix core: even divisors of 61440 in [16, 7680].
 * ------------------------------------------------------------------------------------------ */
/* librosa.stft(n_fft, hop, periodic Hann(n_fft), center=True) of frames 0 .. l-1 of every band and both channels, scattered
 * into the combined spectrogram spec [2][n_rows][l] (complex, re/im interleaved): bins [crop_start, crop_stop) of a band go
 * to rows row0 .. row0 + crop_stop - crop_start, times row_gain[row] (device [n_rows]).  Rows no band covers are left as
 * they are.  bands: host int64 [n_bands][8] = (offset of the band's two rows in wav, L, row pitch ldw, n_fft, hop, crop_start,
 * crop_stop, row0); n_bands <= 4; each band needs 1 + L / hop >= l frames.  zero_pad: edges padded with n_fft/2 zeros
 * (librosa >= 0.9's pad_mode="constant"), else reflected.  high (nullable): bins [high_lo, high_lo + high_h) of band
 * high_band, unscaled, to high [2][high_h][l] (the slice `mirroring` reads). */
int evk_vr_band_stft(const float* wav, const int64_t* bands, int32_t n_bands, int32_t l, const float* row_gain, float* spec,
                     int32_t n_rows, int32_t high_band, int32_t high_lo, int32_t high_h, float* high, int32_t zero_pad,
                     evk_stream_t stream);
/* mag[i] = |spec[i]| / coef over n complex elements, coef = max |spec| written to coef[0] (device).  An all-zero spectrum
 * gives coef 0 and NaN magnitudes, as numpy's 0 / 0.  Max is exact, so the result does not depend on the reduction order. */
int evk_vr_mag_norm(const float* spec, int64_t n, float* mag, float* coef, evk_stream_t stream);
/* scipy.signal.resample_poly's output for a zero-prefixed filter h [nh] (device, the taps times up):
 * y[r][n] = sum_i x[r][i] h[(n + n_pre_remove) down - i up] over the i with that index in [0, nh), ascending i, fp32;
 * n = 0 .. n_out-1.  x [rows][ldx], y [rows][ldy]. */
int evk_resample_poly(const float* x, int32_t rows, int32_t L, int32_t ldx, const float* h, int32_t nh, int32_t up, int32_t down,
                      int32_t n_pre_remove, float* y, int32_t n_out, int32_t ldy, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Normalize.ssl (normalize.py:151-179), the waveform half: loudness normalisation of B zero-padded rows of 32 kHz samples.
 * ------------------------------------------------------------------------------------------ */
enum evk_ssl_status { EVK_SSL_OK = 0, EVK_SSL_SKIP = 1, EVK_SSL_NONFINITE = 2 };
/* Row b of a [B][lda] holds lens[b] (int32 device) samples.  m = max |a| (NaN if a sample is NaN);
 * a32 [B][ld16] = int16((a / m * c1) + c2 * a) and a32b [B][ldb] = (a / m * c1b) + c2b * a with c1 = 0.95 * 0.5 * 32768,
 * c2 = 0.5 * 32768, c1b = 0.95 * 0.5 * 1145.14, c2b = 0.5 * 1145.14 (float64 products rounded to float32), every operation a
 * float32 operation in that order (bit-identical to numpy); the int16 conversion truncates to int32 and keeps the low 16 bits
 * (x86 numpy's astype).  Entries at or past lens[b] are 0.  status[b] (int32 device): EVK_SSL_SKIP if (double)m > 2.2,
 * else EVK_SSL_NONFINITE if m is 0 or NaN (the outputs are then NaN), else EVK_SSL_OK. */
int evk_ssl_normalize(const float* a, int32_t lda, const int32_t* lens, int32_t B, int32_t L, int16_t* a32, int32_t ld16,
                      float* a32b, int32_t ldb, int32_t* status, evk_stream_t stream);
/* Half spectra of every band of both outputs, the input of evk_istft.  From the combined spectrogram x [2][n_rows][l]
 * (complex) and the net's pred [2][n_rows][l] (pred_tta nullable: (pred + pred_tta) * 0.5 * coef, else pred * coef; coef a
 * device scalar): y = pred exp(i angle(x)) (angle(0) = 0), v = x - y.  Band b (host int64 [n_bands][6] = (n_fft,
 * crop_start, crop_stop, row0, offset of its gains in `gains`, offset of its frames in `out` in complex elements)) gets
 * out [4][l][n_fft/2 + 1] complex, rows (y ch0, y ch1, v ch0, v ch1): bin k = gains[k] * (combined row row0 + k - crop_start
 * for k in [crop_start, crop_stop), 0 elsewhere).  With high [2][high_h][l] (nullable), the top band's bins
 * [n_fft/2 - high_h, n_fft/2) are spec_utils.mirroring of the output instead: the flipped magnitudes of its rows
 * [mirror_lo, mirror_lo + high_h) with the phase of high, or high itself where |high| <= that. */
int evk_vr_assemble(const float* x, const float* pred, const float* pred_tta, const float* coef, int32_t n_rows, int32_t l,
                    const float* high, int32_t high_h, int32_t mirror_lo, int32_t top, const int64_t* bands, int32_t n_bands,
                    const float* gains, float* out, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * AudioService.slicer (service/audio.py:142-183; audiokit/slicer/slicer.py), slicer.cu.
 * ------------------------------------------------------------------------------------------ */
/* Slicer.get_rms of B rows: row b of x [B][ldx] holds lens[b] (int32 device) samples.  rms [B][ldr], T <= ldr frames per row:
 * frame t = sqrt(mean(x[t hop - win/2 .. t hop - win/2 + win)^2)) with zeros outside the row, for t < 1 + (lens[b] + 2 (win/2)
 * - win) / hop (1 + lens[b] / hop for even win); later frames are 0.  Squares, sums, mean and root are float64 in a fixed
 * order, rounded to float32 once: within 1 ulp of the exact value, and the same bits for a row alone or in any batch.
 * win <= 64 hop; B <= 65535. */
int evk_frame_rms(const float* x, int64_t ldx, const int32_t* lens, int32_t B, int32_t win, int32_t hop, float* rms, int32_t T,
                  int32_t ldr, evk_stream_t stream);
enum evk_slice_status { EVK_SLICE_OK = 0, EVK_SLICE_SILENT = 1, EVK_SLICE_NONFINITE = 2 };
/* The chunk loop of audio.py:171-178.  chunks: int64 device [n_chunks][2] = (offset in x and y, length), max_len >= every
 * length (host), n_chunks <= 65535.  Per chunk, m = max |x| (NaN if a sample is NaN) is written to m [n_chunks] (device) and
 *   c = m > 1 ? x / m : x;   y = int16(((c / m * c1) + c2 * c) * 32767)
 * to y at the chunk's offsets, every operation a float32 operation in that order (bit-identical to numpy); the int16
 * conversion truncates to int32 and keeps the low 16 bits, NaN and values outside int32 giving 0 (x86 numpy's astype).
 * status [n_chunks] (int32 device): EVK_SLICE_SILENT if m == 0 (every output is int16(NaN) = 0), EVK_SLICE_NONFINITE if m is
 * NaN or Inf, else EVK_SLICE_OK.  Samples outside every chunk are not written. */
int evk_slice_normalize(const float* x, const int64_t* chunks, int32_t n_chunks, int64_t max_len, float c1, float c2, int16_t* y,
                        float* m, int32_t* status, evk_stream_t stream);
/* TTS.audio_postprocess (inference/tts.py:878-907), tts.py.  frags: int64 device [n_frags][2] = (offset in x, length), dst:
 * int64 device [n_frags] = offset in y, max_len >= every length (host), n_frags <= 65535, gap >= 0 (int(sr * interval)).
 * Per fragment, m = max |x| (NaN if a sample is NaN) is written to m [n_frags] (device) and
 *   y[dst + i] = int16((m > 1 ? x[i] / m : x[i]) * 32768)  for i < length,   y[dst + length + j] = 0  for j < gap,
 * float32 operations without contraction, converted as evk_slice_normalize converts: 1.0 gives -32768, as the reference does.
 * Samples of y outside every [dst, dst + length + gap) are not written. */
int evk_fragment_int16(const float* x, const int64_t* frags, const int64_t* dst, int32_t n_frags, int64_t max_len, int64_t gap,
                       int16_t* y, float* m, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Whisper transcription (whisper.py, asr.py), inference only: csrc/whisper.cu.  Token, position and counter arguments
 * named *_dev / pos / gstep are int32 device scalars, so the decode step replays as a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* Whisper's log-mel features of B whole clips of 16 kHz samples: row b of wav [B][ld_wav] holds lens[b] (int32 device,
 * lens[b] >= 201, lens[b] / 160 <= T) samples.  out [B][T][n_mels]: frame t < lens[b] / 160 of row b is the 400-point
 * periodic-Hann STFT (hop 160, centre reflect padding) as a direct DFT against basis = [400][201] window * cos | [400][201]
 * -window * sin, |X|^2 @ fb ([201][n_mels]), log10(max(., 1e-10)), then max(x, clip max - 8) and (x + 4) / 4 with the max
 * over all of the clip's own frames; frames from lens[b] / 160 to T are 0 (padding in the feature domain).  The max is taken
 * per 256 frames into part [B][ceil(T / 256)] and folded in chunk order.  fp32 FMAs in a fixed order: the same bits alone or
 * in any batch, and for any T.  T = 3000 gives the 30 s input of the encoder.  n_mels <= 256, B <= 65535. */
int evk_whisper_logmel(const float* wav, int64_t ld_wav, const int32_t* lens, int32_t B, int32_t T, const float* basis,
                       const float* fb, int32_t n_mels, float* part, float* out, evk_stream_t stream);
/* x[r] = emb[tok[r]] + pe[*pos] for r < R (rows of d floats, contiguous). */
int evk_whisper_embed(const int32_t* tok, const float* emb, const float* pe, const int32_t* pos, int32_t R, int32_t d, float* x,
                      evk_stream_t stream);
/* x[r] += pe[r % T] for the rows < rows of x [rows][d] (contiguous): the encoder's fixed positions. */
int evk_whisper_add_pos(float* x, int64_t rows, int32_t T, int32_t d, const float* pe, evk_stream_t stream);
/* Self-attention cache without per-step copies: row r < R writes its K | V (columns [d, 3d) of qkv [R][ldq]) once, into slot
 * s = r * S + *pos of pool (rows of ld_pool floats, K at 0, V at d), and sets tab[r][*pos] = s (tab [R][ld_tab], S <= ld_tab).
 * A slot is written at most once per decode, so a beam reordering gathers only the tables. */
int evk_whisper_self_kv(const float* qkv, int32_t ldq, int32_t d, float* pool, int64_t ld_pool, int32_t* tab, int32_t ld_tab,
                        const int32_t* pos, int32_t R, int32_t S, evk_stream_t stream);
/* Decode attention, head dim 64, exact fp32 (no tensor cores), softmax(scale q k^T) v per head h < H.  Query row g * nq + a
 * (a < nq) of q [.][ldq]; output o [.][ldo] at the same row.  K of key row k is kv + k * ld_kv + h * 64, V is v_off further.
 *   tab != null (self-attention): nq == 1, the keys of group g are rows tab[g][j], j <= *pos, and *pos < n_keys <= ld_tab;
 *   tab == null (cross-attention): the keys of group g are rows g * n_keys + j, j < n_keys, read once for the group's nq
 *   (<= 8) queries: the beams of a clip share its cross K / V.
 * Each row's result depends only on its own query and keys: the same bits in any batch.  kv 16-byte aligned, ld_kv and v_off
 * multiples of 4; nq * (64 + n_keys) floats of shared memory (<= 200 KB). */
int evk_whisper_attn(const float* q, int32_t ldq, const float* kv, int64_t ld_kv, int32_t v_off, const int32_t* tab,
                     int32_t ld_tab, const int32_t* pos, int32_t n_keys, int32_t groups, int32_t nq, int32_t H, float scale,
                     float* o, int32_t ldo, evk_stream_t stream);
/* y = LayerNorm(x) * gamma + beta over the C floats of each row < rows of x [rows][ldx] (y [rows][ldy], not in place), any C:
 * one row per block, mean and centred variance summed in a fixed order, so a row's bits do not depend on the batch. */
int evk_whisper_layernorm(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, float* y, int32_t ldy,
                          int64_t rows, int32_t C, evk_stream_t stream);
/* The pass at <|startoftranscript|>: per row r < R of logits [R][ld] (V classes), nsp[r] = softmax(row)[nospeech] and
 * lang_tok[r] = the id in lang_ids [n_lang] (device) with the largest logit (the lowest id on a tie). */
int evk_whisper_first_pass(const float* logits, int64_t ld, int32_t R, int32_t V, int32_t nospeech, const int32_t* lang_ids,
                           int32_t n_lang, float* nsp, int32_t* lang_tok, evk_stream_t stream);
/* One beam-search step of transformers' Whisper generate (num_beams = beam <= 8, early_stopping False) for `clips` clips of
 * `beam` rows each (row = clip * beam + b).  *gstep = g, the tokens generated so far; the logits [clips * beam][ld] are those
 * of position plen - 1 + g.  Per row (cand_val / cand_tok [rows][2 beam] scratch): log_softmax; suppress `sup` [n_sup], and
 * `bsup` [n_bsup] when g == 0 (device lists); WhisperTimeStampLogitsProcessor with eot, nots = <|notimestamps|>, tsb = first
 * timestamp, mit = max_initial_timestamp_index (< 0: none); plus run_score[row]; the top 2 beam.  Per clip, as
 * GenerationMixin._beam_search: the top 2 beam of the clip's candidates, the best `beam` non-eot ones become the next rows
 * (tok, parent = source row, run_score), eot hypotheses among the first `beam` (and all at plen + g + 1 == maxlen) enter the
 * finished set (fin_score [clips][beam], score / (g + 1)^length_penalty; fin_seq [clips][beam][ld_hist], fin_len, fin_flag),
 * and unsat[clip] becomes 0 when the running beams can no longer beat it; a clip with unsat == 0 is not touched.  hist
 * [rows][ld_hist] (generated tokens) and tab [rows][ld_tab] (slot tables, entries <= plen - 1 + g) of the new rows are
 * gathered from their parents.  The caller advances *gstep.  Everything stays in device memory.  ld_hist, ld_tab <= 448,
 * maxlen - plen <= ld_hist, maxlen <= ld_tab, V <= 262144.
 * row_lse, run_lse, fin_lse: all null, or all given (anything else is EVK_ERR_ARG) to follow each hypothesis' log-sum-exp of
 * its processed rows: row_lse [rows] (scratch) gets the log-sum-exp of each row's processed log-probs, run_lse [rows] of the
 * new rows is their parent's run_lse + row_lse, and fin_lse [clips][beam] moves with the finished set as fin_score does.  For
 * a finished hypothesis of L tokens, fin_score - fin_lse / L (length_penalty 1) is transformers' long-form avg_logprob: the
 * mean of log_softmax(processed row)[token].  The caller zeroes run_lse and fin_lse before the first step.  Tokens and
 * scores do not depend on whether they are given. */
int evk_whisper_beam_step(const float* logits, int64_t ld, int32_t clips, int32_t beam, int32_t V, int32_t eot, int32_t nots,
                          int32_t tsb, int32_t mit, int32_t plen, int32_t maxlen, const int32_t* sup, int32_t n_sup,
                          const int32_t* bsup, int32_t n_bsup, const int32_t* gstep, float length_penalty, float* cand_val,
                          int32_t* cand_tok, float* run_score, int32_t* hist, int32_t ld_hist, int32_t* tab, int32_t ld_tab,
                          int32_t* tok, int32_t* parent, float* fin_score, int32_t* fin_seq, int32_t* fin_len, int32_t* fin_flag,
                          int32_t* unsat, float* row_lse, float* run_lse, float* fin_lse, evk_stream_t stream);
/* 30 s windows of whole-clip log-mels lm [B][T][n_mels]: output row r < R of out [R][3000][n_mels] is frames
 * [seek, seek + n) of clip row `clip`, zero from n on, with (clip, seek, n) = tab[r][0..2] (int32 device, clip < B,
 * 0 <= seek, n <= 3000).  Frames at or past T read as 0.  n = 0 gives a zero row. */
int evk_whisper_window(const float* lm, int32_t B, int32_t T, int32_t n_mels, const int32_t* tab, int32_t R, float* out,
                       evk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* EVK_H_ */
