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

int evk_init(void);                    /* checks compute capability 10.x, raises smem limits */
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
 * attentions.py:408-416), their data gradients (one call per stride phase), ConvTranspose1d
 * (models.py:460), nn.Linear / 1x1 convs, and the attention GEMMs (attentions.py:243-292).
 * ------------------------------------------------------------------------------------------ */
typedef struct evk_gconv_desc {
  const float* x; float* w; float* y; const float* res; const float* bias;
  const int32_t* in_len; const int32_t* out_len;
  int64_t x_sb, x_sh, w_sb, w_sh, w_sq, y_sb, y_sh, r_sb, r_sh;
  int32_t ldx, ldw, ldy, ldr;
  int32_t b_sh;          /* bias offset per inner-batch index h (grouped convs run as H = groups) */
  int32_t Z, H;          /* batch count and inner (head) count: b = z / H, h = z % H */
  int32_t C, N, Q, G;    /* in-channels, out-channels, taps, groups (G>1: direct kernels only) */
  int32_t Tin, J, P;     /* input positions per batch, output positions computed, inner width */
  int32_t is, os, o0;    /* input stride, output stride, output origin (in positions) */
  int32_t Tout;          /* output positions per batch (bounds for (o0 + j*os)) */
  int32_t act; float slope;
  int32_t off[EVK_MAX_TAPS];
  /* optional fused dropout AFTER the activation (forward launches taken by gemm_tma_kernel only; any other route returns
   * EVK_ERR_UNSUPPORTED): y = dropout_p(act(...)); rng = device [seed, offset] (the library's RNG state), sid = stream id. */
  const uint64_t* drop_rng; uint64_t drop_sid; float drop_p;
} evk_gconv_desc;

int evk_gconv_fwd(const evk_gconv_desc* d, evk_stream_t stream);
int evk_gconv_desc_size(void);         /* sizeof(evk_gconv_desc) as compiled: bindings check their mirror against it */
/* 0 (default): one TF32 product per MAC.  1: 3xTF32 error-compensated products (~fp32 accuracy, 3x tensor work);
 * the parity tests use it to separate indexing errors from TF32 operand rounding. Process-wide. */
int evk_set_precise(int32_t on);
int evk_get_precise(void);
/* 1 (default): eligible launches run on the wgmma kernels (gemm_tma.cu, gconv_tc.cu); 0: mma.sync kernels only. */
int evk_set_backend(int32_t tensor_core);
/* Dispatch accounting: algorithmic flops enqueued since the last reset, per kernel family (host-side counters; graph
 * replays add nothing).  out[i], i < EVK_DISPATCH_SLOTS:
 *   0 conv/linear fwd-like on gemm_tma_kernel (TMA + wgmma)   1 ... on gconv_tc_kernel (wgmma, staged slab)
 *   2 ... on gconv_f_kernel (mma.sync)                          3 ... on the direct CUDA-core kernels
 *   4 weight gradients on gemm_tma_kernel                        5 ... on gconv_w_kernel (mma.sync)
 *   6 ... on the direct kernels                                  7 plain evk_gemm_tf32 calls */
/* A/B switches of gemm_tma_kernel: slab (default 1) = stride-1 tap sums stage one input slab per channel block and run every
 * tap from it; mt2 (default 1) = 256-row tiles where the persistent grid's wave quantisation allows; trunc_comp (default
 * 3.52e-4) = accumulator compensation per raw fp32 operand for the tensor core's TF32 operand truncation (0 disables). */
int evk_set_tma_options(int32_t slab, int32_t mt2, float trunc_comp);
#define EVK_DISPATCH_SLOTS 8
int evk_dispatch_stats(double* out, int32_t n);
int evk_dispatch_stats_reset(void);
/* Weight gradient of the same operator:  W[z][q][n][c] += sum_{j,w} Yg[z][orow][n] * X[z][irow][c]
 * (d->y is read as the output gradient, d->w is accumulated -- partial sums added in a fixed order, so the result is
 * reproducible; when w_sb == w_sh == 0 the
 * sum also runs over z).  Replaces autograd's conv weight-gradient kernels for the call sites above. */
int evk_gconv_wgrad(const evk_gconv_desc* d, evk_stream_t stream);
/* Direct (CUDA-core) variants for skinny layers: C/G < 8 (1-channel inputs, grouped k=41 convs of
 * DiscriminatorS, models.py:563-575).  Same descriptor; W is [Q][N][C/G]. */
int evk_conv_direct_fwd(const evk_gconv_desc* d, evk_stream_t stream);
int evk_conv_direct_dgrad(const evk_gconv_desc* d, evk_stream_t stream);  /* d->x is WRITTEN (dX), d->y read */
int evk_conv_direct_wgrad(const evk_gconv_desc* d, evk_stream_t stream);

/* out[n] (+)= sum_rows x[row][n]  -- bias gradients */
int evk_colsum(const float* x, int64_t rows, int32_t n, int32_t ld, float* out, int32_t accumulate, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Weight preparation: torch.nn.utils.weight_norm (modules.py:154-171, models.py:425-435,489-587)
 * folded into the operand-packing pass.  v is [D0][D1][Q] (torch layout), g is [D0] or NULL
 * (plain weight).  Produces PA[q][d0][d1] (pitch lda) and optionally PB[q][d1][d0] (pitch ldb).
 * ------------------------------------------------------------------------------------------ */
int evk_weight_pack(const float* v, const float* g, int32_t D0, int32_t D1, int32_t Q, float* pa, int32_t lda,
                    float* pb, int32_t ldb, evk_stream_t stream);
/* Same, with the channel dims zero-padded to D0p x D1p rows/cols (PA is [Q][D0p][lda], PB [Q][D1p][ldb], both
 * pre-zeroed by the caller): 1-channel layers are padded to 4 so they run on the tensor-core kernels. */
int evk_weight_pack_p(const float* v, const float* g, int32_t D0, int32_t D1, int32_t Q, float* pa, int32_t lda,
                      int32_t D0p, float* pb, int32_t ldb, int32_t D1p, evk_stream_t stream);
int evk_weight_pack_bwd_p(const float* dpa, int32_t lda, int32_t D0p, const float* v, const float* g, int32_t D0,
                          int32_t D1, int32_t Q, float* dv, float* dg, evk_stream_t stream);
/* given dPA (gradient in PA layout) -> dv [D0][D1][Q] (written), dg [D0] (written) (g may be NULL) */
/* Whole-network variants (pack_batched.cu): ONE launch packs / back-propagates every weight of a network.  `jobs` is a
 * device array of 88-byte records {v, g, pa, pb, dpa, dv, dg (pointers); D0, D1, Q, lda, D0p, ldb, D1p, row0 (int32)},
 * job_of_row [nrows] maps each (job, output-channel) row to its job.  All pointers are static arenas owned by the caller. */
int evk_weight_pack_batched(const void* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream);
int evk_weight_pack_bwd_batched(const void* jobs, const int32_t* job_of_row, int32_t nrows, evk_stream_t stream);
int evk_weight_pack_bwd(const float* dpa, int32_t lda, const float* v, const float* g, int32_t D0, int32_t D1,
                        int32_t Q, float* dv, float* dg, evk_stream_t stream);

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
/* General STFT (stft.cu): n_fft in {256..4096} (power of two), any hop, power-of-two win <= n_fft (periodic Hann, centred in
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
 * * gamma[c] + beta[c], biased variance; optional exact GELU applied to the result (act_gelu != 0).  Forward only. */
int evk_instnorm_cl(const float* x, int32_t ldx, const float* gamma, const float* beta, float eps, int32_t act_gelu, float* y,
                    int32_t ldy, int32_t B, int32_t T, int32_t C, evk_stream_t stream);
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
/* dS = P * (dP - sum_j dP*P) * scale, in place on dP; also emits drelk[z][i][r] = dS[i][i+r-win] (nullable) */
int evk_attn_softmax_bwd(const float* P, float* dP, int32_t lds, int32_t Z, int32_t Tq, int32_t Tk, float scale, float* drelk,
                         int32_t win, evk_stream_t stream);
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
/* Weight gradient of a stride-1 (dilated, period-folded) conv on the same kernel:
 *   dW[q][n][c] += sum_b sum_pos dY[b][pos][n] * X[b][pos + off[q]*P][c]
 * on operands transposed by evk_transpose_rows (contraction index contiguous): dyt [B][N][ld_dy] (out_rows = J*P valid),
 * xt [4][B][C][ld_x] with pitch x_rs between four copies delayed by r = 0..3 positions, xt_r[b][c][u] = X[b][u - r][c]
 * (in_rows + r valid, evk_transpose_rows with shift = r).  TMA coordinates along the contiguous dimension must be 16-byte
 * aligned: a tap shift s reads copy r = (-s) mod 4 at the aligned offset s + r; only the copies that occur need filling.  Rows outside the input (the conv padding) are zero-filled by the copy engine.
 * Accumulates the K splits' partials, added in split order, into dW (pitch ldw, tap pitch w_sq); off is a HOST array. */
int evk_conv_wgrad_tma(const float* dyt, int32_t ld_dy, int64_t dy_sb, const float* xt, int32_t ld_x, int64_t x_sb, int64_t x_rs, float* dW,
                       int32_t ldw, int64_t w_sq, int32_t B, int32_t N, int32_t C, int32_t out_rows, int32_t in_rows,
                       int32_t Q, int32_t P, const int32_t* off, int32_t splits, evk_stream_t stream);
/* Everything a conv's backward needs from its output gradient in one pass (elementwise.cu): g = dy * act'(y) * (t < len*P);
 * dpre (nullable) = g in the layout of dy; dyt (nullable) [B][C][ldt] = g transposed (the K-major operand of evk_conv_wgrad_tma);
 * dbias (nullable, [C], zero-initialised by the caller) += column sums of g.  act: evk_act of the forward epilogue, yact = its
 * OUTPUT (derivatives are taken from the output: leaky-ReLU / ReLU by sign, tanh by 1 - y^2). */
int evk_dy_prep(const float* dy, int32_t lddy, const float* yact, int32_t ldy, int32_t act, float slope, float gscale, const int32_t* len,
                int32_t P, float* dpre, int32_t ldp, float* dyt, int32_t ldt, int64_t t_sb, float* dbias, int32_t B, int32_t T, int32_t C,
                evk_stream_t stream);
/* gscale multiplies g: 1/(1-p) when the forward epilogue applied dropout after a ReLU -- the saved OUTPUT is then zero exactly
 * where the element was dropped or the ReLU was off, so no mask needs to be regenerated. */
/* Strided conv forward on the same kernel: the input is first split into `stride` phase copies
 *   xs[rho][b][j*P + w][c] = x[b][(j*stride + rho)*P + w][c]   (zero for j*stride + rho >= T; j < Jp = ceil(T / stride))
 * and the conv becomes a stride-1 tap sum in which tap q (u = q*dil - pad) reads copy src[q] = u mod stride at row shift
 * off[q] = floor(u / stride).  d describes that stride-1 form (d->x = copy 0, d->Tin = Jp, d->is = 1, d->off = shifts);
 * copies are x_ps floats apart; src is a HOST array.  Returns EVK_ERR_UNSUPPORTED if the launch is not eligible. */
int evk_phase_split(const float* x, int32_t ldx, int64_t x_sb, float* xs, int64_t xs_ps, int32_t B, int32_t T, int32_t P,
                    int32_t C, int32_t stride, int32_t Jp, evk_stream_t stream);
int evk_gconv_fwd_phased(const evk_gconv_desc* d, int32_t phases, int64_t x_ps, const int32_t* src, evk_stream_t stream);
/* [B][T][ldx] (C valid, batch pitch x_sb) -> [B][C][ldy] (T + shift valid, batch pitch y_sb):
 * y[b][c][u] = x[b][u - shift][c], zero for u < shift. */
int evk_transpose_rows(const float* x, int32_t ldx, int64_t x_sb, float* y, int32_t ldy, int64_t y_sb, int32_t B, int32_t T,
                       int32_t C, int32_t shift, evk_stream_t stream);
/* every delayed copy r (bit r of mask, r = 0..3) in one pass over x: y[r*y_rs + ...][b][c][u] = x[b][u - r][c]. */
int evk_transpose_rows_multi(const float* x, int32_t ldx, int64_t x_sb, float* y, int32_t ldy, int64_t y_sb, int64_t y_rs,
                             int32_t B, int32_t T, int32_t C, int32_t mask, evk_stream_t stream);

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
 * batch size).  rows <= 4 requires rows_rounded_up_to_a_power_of_2 * C <= 10240.  act: EVK_ACT_NONE / RELU / LRELU. */
int evk_gemv_rows(const float* x, int32_t ldx, int32_t rows, const float* W, int32_t ldw, const float* bias, float* y,
                  int32_t ldy, int32_t N, int32_t C, int32_t act, float slope, evk_stream_t stream);
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
/* Fused token sampler of batched KV-cache decoding (infer_panel_batch_infer, t2s_model.py:563-730; utils.py:109-157), one CTA
 * per row b of logits [B][ldl] (V <= 2048 classes, eos = V - 1), in the reference's order: repetition penalty over the row's
 * history (prompt included) -> top-p if top_p < 1 (descending order, cumulative softmax, `cum > top_p` removed, the first kept;
 * on the penalised, un-tempered logits) -> / max(T, 1e-5) -> top-k (values >= the k-th largest kept) -> softmax ->
 * argmax(p / q), q ~ Exp(1).  The step is idx = *n_dev - icfg[2]; at idx 0 EOS is excluded.  The row stops when the token or the
 * argmax of the penalised logits is EOS (fin[b] = (idx, idx - 1)), else when idx + 1 > early_stop (!= -1) or idx == max_steps - 1
 * (fin[b] = (idx, idx)); a row with fin[b][0] >= 0 is left untouched.  Otherwise hist[b][prefix + idx] = token, its bit is set
 * in seen, and x_next[b] = emb[token] + alpha[0] * pe[prefix + idx].
 *   icfg: device int64 [6] = (seed, prefix, n0, top_k >= 1, early_stop, max_steps);  fcfg: device float [3] = (top_p, T, penalty)
 *   q: NULL (counter-based Exp(1) draws keyed by (seed, row, idx, class)) or supplied draws [B][ldq]
 *   hist: int64 [B][ldh];  seen: uint32 [B][(V + 31) / 32] bitmap of the tokens in hist;  fin: int32 [B][2], -1 while running
 *   emb: [V][D], pe: [*][D], x_next: [B][D]. */
int evk_sample_tokens(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, const int64_t* icfg,
                      const float* fcfg, const int32_t* n_dev, const float* q, int32_t ldq, int64_t* hist, int32_t ldh,
                      uint32_t* seen, int32_t* fin, const float* emb, const float* pe, const float* alpha, float* x_next,
                      int32_t D, evk_stream_t stream);
/* The same with EOS excluded at every step idx < eos_steps (>= 0) instead of at step 0 only: evk_sample_tokens is this call with
 * eos_steps = 1.  infer_panel_naive (t2s_model.py:835-836) passes 11, with a prompt or without one (prefix 0). */
int evk_sample_tokens_ex(const float* logits, int32_t ldl, int32_t B, int32_t V, int32_t eos, int32_t eos_steps,
                         const int64_t* icfg, const float* fcfg, const int32_t* n_dev, const float* q, int32_t ldq, int64_t* hist,
                         int32_t ldh, uint32_t* seen, int32_t* fin, const float* emb, const float* pe, const float* alpha,
                         float* x_next, int32_t D, evk_stream_t stream);
int evk_ce_fwd(const float* logits, int32_t ld, const int64_t* targets, int32_t rows, int32_t V, int32_t topk,
               int64_t ignore_index, float* lse, float* nll, uint8_t* flags, float* out2, evk_stream_t stream);
int evk_ce_bwd(const float* logits, int32_t ld, const int64_t* targets, const float* lse, const float* gscale,
               int32_t rows_per_g /* row r is scaled by gscale[r / rows_per_g]; == rows for one scalar */, float* dl,
               int32_t lddl, int32_t rows, int32_t V, evk_stream_t stream);
/* DPO head of Text2SemanticDecoder.forward (t2s_model.py:393-429; utils.py:160-192 with reference_free=True): from the
 * per-token nll of the chosen [B, Yc] and rejected [B, Yr] sequences: out3 = (sum CE of chosen, mean_b -logsigmoid(beta *
 * (logp_chosen_b - logp_rejected_b)), their sum); coef_c/coef_r [B] = d out3[2] / d nll_{c,r}[b][t] (feeds evk_ce_bwd). */
int evk_dpo_head(const float* nll_c, int32_t Yc, const float* nll_r, int32_t Yr, int32_t B, float beta, float* out3,
                 float* coef_c, float* coef_r, evk_stream_t stream);
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
 * o: [B, L, ldo].  Requires 1 <= lens[b] <= L <= 512 (lens: int64 device [B], values outside are clamped to [1, L]),
 * ld % 4 == 0, ldo % 2 == 0, q/k/v 16-byte and o 8-byte aligned.  Query rows at or past lens[b] are computed like any
 * other (finite).  Scores are never materialised (online softmax); TF32 mma.sync with fp32 accumulation (3xTF32 under
 * evk_set_precise(1)); no atomics, bit-reproducible. */
int evk_attn_pad_fwd(const float* q, const float* k, const float* v, int32_t ld, float* o, int32_t ldo, int32_t B,
                     int32_t H, int32_t L, const int64_t* lens, float scale, evk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * UVR5 VR separation (CascadedASPPNet and the DeEcho / DeReverb CascadedNet, uvr5.py), inference only.  Activations are
 * channels-last fp32: pixel (b, y, x) of an operand starts at  p + b*bs + (y*W + x)*pitch  (floats), so a channel slice of
 * a concat buffer is an operand.
 * ------------------------------------------------------------------------------------------ */
enum evk_conv2d_act { EVK_C2_NONE = 0, EVK_C2_RELU = 1, EVK_C2_LRELU = 2 /* slope 0.01 */, EVK_C2_SIGMOID = 3 };
/* y = act(conv2d(x, w) * scale[n] + bias[n])  (scale / bias may be null: 1 / 0).  x: [B, H, W, C] (pitch x_pitch >= C,
 * batch stride x_bs); w: [N][k][k][C] (k = 1 or 3); stride 1 or 2, zero padding pad, dilation dil >= 1; y: [B, Ho, Wo, N]
 * (pitch y_pitch >= N, batch stride y_bs), Ho = (H + 2 pad - dil (k - 1) - 1) / stride + 1.  Implicit GEMM with TF32
 * products and fp32 accumulation: wgmma when C, x_pitch and x_bs are multiples of 4 and x, w are 16-byte aligned,
 * mma.sync otherwise and for 3xTF32 under evk_set_precise(1).  No atomics, and every output's sum has one order whatever
 * B is, so results are bit-reproducible and independent of the batch. */
int evk_conv2d_fwd(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, const float* scale, const float* bias,
                   float* y, int32_t y_pitch, int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t N, int32_t k,
                   int32_t stride, int32_t pad, int32_t dil, int32_t act, evk_stream_t stream);
/* evk_conv2d_fwd with zero padding and dilation per axis (the DeEcho / DeReverb ASPP: dilation (4, 2), (8, 4), (12, 6)):
 * Ho = (H + 2 pad_h - dil_h (k - 1) - 1) / stride + 1, Wo likewise with pad_w, dil_w.  Same kernels, dispatch and
 * guarantees; evk_conv2d_fwd(..., pad, dil, ...) is this call with pad_h = pad_w = pad, dil_h = dil_w = dil. */
int evk_conv2d_fwd_hw(const float* x, int32_t x_pitch, int64_t x_bs, const float* w, const float* scale, const float* bias,
                      float* y, int32_t y_pitch, int64_t y_bs, int32_t B, int32_t H, int32_t W, int32_t C, int32_t N,
                      int32_t k, int32_t stride, int32_t pad_h, int32_t pad_w, int32_t dil_h, int32_t dil_w, int32_t act,
                      evk_stream_t stream);
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
/* Inverse of evk_stft_fwd's center=True transform with the periodic Hann(n_fft) window: torch.istft(n_fft, hop, n_fft, hann,
 * center=True, normalized=False, onesided=True, length=None) of cplx [B*S*T][n_fft/2+1][2] (rows b*S + s), times mask when
 * given (bs_roformer.py:530-543): bin k of row (b, s), frame t is multiplied by the complex mask at columns
 * 2 (k S + s) .. +1 of mask row b*T + t (pitch ld_mask: the mask estimator's 'b t (f s c)' layout).  Per frame a C2R inverse
 * DFT (imaginary parts of bins 0 and n_fft/2 ignored) and the window, written to work [B*S*T][n_fft]; then the overlap-add in
 * frame order, divided by the sum of squared windows, trimmed by n_fft/2 at both ends: out [B*S][ld_out] gets hop*(T-1)
 * samples per row.  n_fft a power of two in [256, 4096], T >= 2, hop <= n_fft / 2, B*S <= 65535. */
int evk_istft(const float* cplx, const float* mask, int32_t ld_mask, int32_t B, int32_t S, int32_t T, int32_t n_fft, int32_t hop,
              float* work, float* out, int32_t ld_out, evk_stream_t stream);
/* Band-split operand (bs_roformer.py:481-490 and each band's RMSNorm before its Linear): from evk_stft_fwd's cplx
 * [B*S*T][n_bins][2] (rows b*S + s) to y [B*T][ld_y], row (b, t), column (f S + s) * 2 + c ('b t (f s c)'), with the columns
 * [2 S band_off[i], 2 S band_off[i+1]) of band i divided by max(their L2 norm, 1e-12).  band_off: device int32
 * [n_bands + 1] bin offsets (band_off[n_bands] = n_bins).  S = 1 or 2; 2 S n_bins floats must fit 48 KB. */
int evk_bs_band_input(const float* cplx, int32_t B, int32_t S, int32_t T, int32_t n_bins, const int32_t* band_off,
                      int32_t n_bands, float* y, int32_t ldy, evk_stream_t stream);
/* y[r] = x[r] / max(||x[r]||_2, 1e-12) per row (F.normalize(dim=-1): the RMSNorms, whose gamma * sqrt(dim) the caller folds
 * into the next Linear's weight columns). */
int evk_row_l2norm(const float* x, int32_t ldx, float* y, int32_t ldy, int64_t rows, int32_t C, evk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* EVK_H_ */
