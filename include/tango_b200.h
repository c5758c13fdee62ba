/* tango_b200.h — C ABI of libtango_b200.so (H100 / sm_90a kernels for the Tango inference hot path).
 *
 * The reference (declare-lab/tango) is pure Python on stock PyTorch ops: it has no FFI layer of its own.
 * Each entry point below therefore replaces a *library op call site* of the reference hot path (SURVEY.md §2.1,
 * §8a); the file:line cited is the reference code whose arithmetic the kernel reproduces. The Python host
 * (tango_b200/*.py) binds these with ctypes and mirrors the reference's module interface on top.
 *
 * Conventions: plain pointers (device memory unless stated), explicit sizes/strides, `stream` is a
 * cudaStream_t passed as void*. Every function returns 0 on success and a negative TNG_E* code on error;
 * tng_last_error() gives a message. Nothing is allocated or retained by the library. No CPU fallback exists:
 * without a CUDA device every compute entry point fails with TNG_ECUDA.
 *
 * Activations are channels-last ("NHWC", rows = pixels / tokens / time positions, channels contiguous).
 */
#ifndef TANGO_B200_H
#define TANGO_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define TNG_OK 0
#define TNG_EINVAL (-1) /* bad argument / unsupported shape */
#define TNG_ECUDA (-2)  /* CUDA runtime / driver error (incl. no device) */

#define TNG_ACT_NONE 0
#define TNG_ACT_SILU 1
#define TNG_ACT_LRELU 2 /* slope = act_param */
/* out[j] = (acc[j] + bias[j]) * gelu_erf(acc[j + BN/2] + bias[j + BN/2]) within each N tile of BN columns (weights
 * and bias pre-interleaved), written at output column tn * BN/2 + j. tng_conv_gemm only: BN = block_n (0 = auto) must be
 * 128 or 256 and divide Ncols; bf16 output only (no out_f32, res or rowvec), 16-byte aligned, and alpha = 1. */
#define TNG_ACT_GEGLU 3
#define TNG_ACT_GEGLU_TANH 4 /* same pairing with the tanh-form GELU ("gelu_new": T5 v1.1 gated feed-forward) */

#define TNG_DT_F32 0
#define TNG_DT_BF16 1

#define TNG_MAX_AVIEWS 4
#define TNG_MAX_KGROUPS 40

int tng_version(void);
const char* tng_last_error(void);
/* Number of kernels this library has launched since load (bench.py's `gpu_launches`). */
uint64_t tng_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * tng_conv_gemm — wgmma implicit-GEMM convolution / linear layer (one persistent kernel, TMA-fed).
 * Replaces: nn.Conv2d in ResnetBlock2D / Down/Upsample2D / conv_in / conv_out
 *             (mustango/diffusers/src/diffusers/models/resnet.py:570,590,157,206; unet_2d_condition.py:626,702),
 *           nn.Linear in Transformer2DModel / Attention / GEGLU FeedForward
 *             (transformer_2d.py:255-263,282-290; attention_processor.py:500-540; attention.py:384-387,431-433),
 *           VAE decoder Conv2d (audioldm/variational_autoencoder/modules.py:155-175,658-680),
 *           HiFi-GAN Conv1d / ConvTranspose1d-as-GEMM (audioldm/hifigan/models.py:96-103,124-135,149-165).
 *
 * D[row, n] = sum_g sum_{k<64*nkb_g} A_{view_g}[pixel(row) + (dw_g, dh_g), a_c0_g + k] * B[n, b_k0_g + k]
 *   rows enumerate the output pixel grid (img, h, w), w fastest; A views are bf16 channels-last 4-D tensors
 *   read through TMA with zero fill outside [0,W)x[0,H)x[0,NB) (this is the conv zero padding);
 *   B is a bf16 row-major [Ncols, Ktot] matrix (K contiguous).
 * Epilogue: x = (acc + bias[n] + rowvec[img, n] + res[row, n]) * alpha (+ out_f32[row, n] if accumulate);
 *   out_f32[row, n] = x (optional); out_bf16[row, n] = act(x) (optional; with `split_off > 0` the bf16
 *   rounding residual is also written at column n + split_off — "hi/lo" operand for the 3-term split GEMM).
 */
typedef struct {
  const void* ptr;      /* bf16, element (img, h, w, c) at ptr + img*s_n + h*s_h + w*s_w + c (strides in elements) */
  int64_t C, W, H, NB;  /* extents */
  int64_t s_w, s_h, s_n;
} tng_aview;

typedef struct {
  int32_t view;  /* index into a[] */
  int32_t a_c0;  /* first channel of A */
  int32_t dw, dh; /* tap offset added to the output pixel coordinate */
  int32_t b_k0;  /* first K column of B */
  int32_t nkb;   /* number of 64-wide K blocks */
} tng_kgroup;

typedef struct {
  tng_aview a[TNG_MAX_AVIEWS];
  int32_t n_aviews;
  const void* b; /* bf16 [Ncols, Ktot], row stride ldb elements */
  int64_t Ncols, Ktot;
  int64_t ldb;         /* 0 = Ktot */
  int32_t W, H, NB; /* output pixel grid */
  tng_kgroup g[TNG_MAX_KGROUPS];
  int32_t n_groups;
  /* epilogue */
  const float* bias;   /* [Ncols] or NULL */
  const float* rowvec; /* [NB, rowvec_ld] per-image vector (first Ncols entries used) or NULL */
  int64_t rowvec_ld;   /* 0 = Ncols */
  const void* res;     /* [rows, ldr] residual or NULL */
  int32_t res_dtype;   /* TNG_DT_* */
  int64_t ldr;
  float alpha;
  int32_t accumulate;  /* out_f32 += x */
  float* out_f32;      /* or NULL */
  int64_t ld_f32;
  void* out_bf16;      /* or NULL */
  int64_t ld_bf16;
  int32_t act;         /* TNG_ACT_* applied to the bf16 output only */
  float act_param;
  int32_t split_off;   /* 0 = off */
  int32_t block_n;     /* N tile: 0 = auto; one of 32, 64, 128, 160, 256 */
  /* GroupNorm statistics of the output for the norm that consumes it (resnet.py:555,581; transformer_2d.py:253):
   * gn_stats[(img * Ncols + n) * 2 + {0, 1}] += sum / sum of squares of x[:, n] (the stored value: the fp32 output, or
   * without one the bf16 output, which must then be plain: no activation, no hi/lo split) over the stats_hw rows of image
   * img = row / stats_hw (fp64 accumulators the caller zeroes; per CHANNEL, so that any grouping - also across the
   * channel concat of a skip connection - is a sum of entries). Emitted from the epilogue of the producing GEMM when
   * every tile is full, otherwise by a pass over the output that follows it in the stream, which needs Ncols % 4 == 0
   * and a stored output with ld % 4 == 0 at an 8-byte aligned address (TNG_EINVAL before any launch otherwise).
   * NULL = off. */
  double* gn_stats;
  int64_t stats_hw;
} tng_gemm_desc;

int tng_conv_gemm(const tng_gemm_desc* d, void* stream);
/* What tng_conv_gemm would do with this descriptor, without launching: the N tile, the M tile in `mode` (128, or 256
 * for large non-GEGLU launches at block_n 160; one CTA per SM on mode x block_n tiles) and the split-K factor. Used by
 * bench.py to label its per-kernel timings with the instantiation that actually runs. Any output pointer may be NULL. */
int tng_gemm_plan(const tng_gemm_desc* d, int32_t* block_n, int32_t* mode, int32_t* ksplit);

/* ---------------------------------------------------------------------------------------------------------
 * tng_attention — wgmma flash attention, head width 64, fp32 online softmax.
 * Replaces: Attention + AttnProcessor(2_0) core  softmax(q k^T * scale + bias) v
 *           (mustango/diffusers/src/diffusers/models/attention_processor.py:232-261,263-299,500-540)
 *           and the additive mask bias of unet_2d_condition.py:575-579.
 * q: bf16 rows = batch*Lq tokens, head h at columns q_col0 + 64*h; k, v likewise with Lk tokens per batch.
 * kbias: optional fp32 [batch, Lk] additive bias (already (1-mask)*-10000). out: bf16 [batch*Lq, ld_o],
 * head h at columns 64*h (hi) and, if split_off > 0, the rounding residual at + split_off.
 * nsplit = 1: plain bf16 operands. nsplit = 2: every operand also carries its bf16 rounding residual ("lo") at
 * column + *_lo_off, and the kernel evaluates the 3-term split products hi*hi + lo*hi + hi*lo (parity mode).
 */
typedef struct {
  const void* q; int64_t ld_q; int32_t q_col0; int32_t q_lo_off;
  const void* k; int64_t ld_k; int32_t k_col0; int32_t k_lo_off;
  const void* v; int64_t ld_v; int32_t v_col0; int32_t v_lo_off;
  const float* kbias;
  void* out; int64_t ld_o; int32_t split_off;
  int32_t batch, heads, Lq, Lk;
  float scale;
  int32_t nsplit;
} tng_attn_desc;

int tng_attention(const tng_attn_desc* d, void* stream);

/* tng_attention_wide — wgmma flash attention for ONE head of width `dim` = 512, Lq = Lk = L, no mask: the AudioLDM VAE
 * AttnBlock  softmax(q k^T * scale) v  over the H*W positions of each image
 * (audioldm/variational_autoencoder/modules.py:204-230). q / k / v: bf16 rows = batch*L positions, the operand at columns
 * [col0, col0 + dim) of a row-major matrix with leading dimension ld (elements); out: bf16 [batch*L, ld_o], columns
 * [0, dim). The [L, L] score matrix stays on the SM (S, P and O live in registers). L must be a multiple of 128. */
int tng_attention_wide(const void* q, int64_t ld_q, int32_t q_col0, const void* k, int64_t ld_k, int32_t k_col0,
                       const void* v, int64_t ld_v, int32_t v_col0, void* out, int64_t ld_o, int32_t batch, int32_t L,
                       int32_t dim, float scale, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * GroupNorm (+SiLU) over channels-last input that may be the channel concat of two tensors (skip connection).
 * Replaces: nn.GroupNorm + SiLU in ResnetBlock2D (resnet.py:555-557,581-587), conv_norm_out
 *           (unet_2d_condition.py:699-701), Transformer2DModel.norm (transformer_2d.py:253),
 *           torch.cat skip (unet_2d_blocks.py:2210,2495), VAE Normalize+swish (modules.py:37-41,155-175).
 * Statistics are kept PER CHANNEL: col_stats fp64 [NB, C, 2] (sum, sum of squares over the HW pixels of an image). They
 * normally come out of the producing tng_conv_gemm (gn_stats above); tng_groupnorm_stats is the stand-alone pass for
 * tensors no GEMM produced (it ADDS to col_stats: the caller zeroes them).
 */
int tng_groupnorm_stats(const void* x, int32_t dt, int64_t C, int64_t ld, int64_t NB, int64_t HW, double* col_stats,
                        void* stream);
/* y = act((x - mean) * rstd * gamma + beta) -> bf16 [NB*HW, ld_y] (+ lo half at split_off if > 0) for x = [x0 | x1]
 * (x1 / stats1 may be NULL); mean / rstd of group g over its (C0 + C1) / groups consecutive channels of the concat, from
 * stats0 [NB, C0, 2] and stats1 [NB, C1, 2]; optional bf16 copy of the *raw* concat input to raw_bf16 (the operand of
 * the fused 1x1 shortcut conv). */
int tng_groupnorm_apply(const void* x0, int32_t dt0, int64_t C0, const double* stats0, const void* x1, int32_t dt1,
                        int64_t C1, const double* stats1, int64_t NB, int64_t HW, int32_t groups, const float* gamma,
                        const float* beta, float eps, int32_t act, void* y, int64_t ld_y, int32_t split_off,
                        void* raw_bf16, int64_t ld_raw, int32_t raw_split_off, void* stream);

/* LayerNorm over the last dim of fp32 [rows, C] -> bf16 (attention.py:259,267,274). */
int tng_layernorm(const float* x, int64_t rows, int64_t C, const float* gamma, const float* beta, float eps,
                  void* y, int64_t ld_y, int32_t split_off, void* stream);

/* ---- text-conditioning front-end (SURVEY.md section 8(f).1): FLAN-T5 encoder as called from models.py:98-100 (T5EncoderModel),
 * models.py:129-147 (encode_text) and models.py:266-305 (encode_text_classifier_free). The arithmetic lives in the pip
 * dependency `transformers` (models/t5/modeling_t5.py: T5LayerNorm, T5Attention, T5DenseGatedActDense, T5Stack), which is
 * not under /root/reference; the entry points below replace those modules, the projections run through tng_conv_gemm. */

/* T5LayerNorm: y = x * rsqrt(mean(x^2) + eps) * gamma over the last dim of fp32 [rows, C] -> bf16 y (+ lo half) and/or a
 * dense fp32 copy y_f32 [rows, C] (the final_layer_norm output handed to the UNet); either output may be NULL. */
int tng_rmsnorm(const float* x, int64_t rows, int64_t C, const float* gamma, float eps, void* y, int64_t ld_y,
                int32_t split_off, float* y_f32, void* stream);
/* nn.Embedding lookup (T5Stack.embed_tokens): out[r, :] = table[ids[r], :], fp32 [rows, C]; ids are int64 and must lie in
 * [0, n_table_rows) (checked by the caller, as nn.Embedding's own index check is host-side on CPU). */
int tng_gather_rows(const float* table, int64_t n_table_rows, const int64_t* ids, int64_t rows, int64_t C, float* out,
                    void* stream);
/* T5Attention.forward core for head width 64: softmax(q k^T + relbias[h, key - query] + kbias[b, key]) v, no score
 * scaling. qkv: fp32 [batch*L, ld] with the q / k / v blocks of `heads*64` columns at q_col0 / k_col0 / v_col0;
 * relbias: fp32 [heads, 2L-1] (index key - query + L - 1; the bucketed relative_attention_bias of block 0, shared by all
 * blocks); kbias: fp32 [batch, L] additive key mask (0 or finfo.min, as get_extended_attention_mask builds it) or NULL;
 * out: bf16 [batch*L, ld_o] (+ lo half at split_off). */
int tng_rel_attention(const float* qkv, int64_t ld, int32_t q_col0, int32_t k_col0, int32_t v_col0, int32_t batch,
                      int32_t heads, int32_t L, const float* relbias, const float* kbias, void* out, int64_t ld_o,
                      int32_t split_off, void* stream);

/* fp32 [rows, C] -> bf16 [rows, ld_y] with optional activation, optional hi/lo split, optional nearest x2
 * upsample of an (NB, H, W) grid (resnet.py:146; modules.py:53-57) — the cast in front of a conv that consumes
 * the residual stream directly (conv_in, Downsample2D, Upsample2D, HiFi-GAN leaky_relu -> conv). */
int tng_cast_act(const float* x, int64_t NB, int64_t H, int64_t W, int64_t C, int64_t ld_x, int32_t upsample2x,
                 int32_t act, float act_param, void* y, int64_t ld_y, int32_t split_off, void* stream);

/* Row softmax of fp32 [rows, L] * scale -> bf16 [rows, ld_y] (VAE AttnBlock, modules.py:211-214). */
int tng_softmax_rows(const float* x, int64_t rows, int64_t L, int64_t ld_x, float scale, void* y, int64_t ld_y,
                     int32_t split_off, void* stream);

/* bf16 [B, R, C] -> bf16 [B, C, R] (per-batch transpose; builds K-major V^T for the VAE attention PV GEMM). */
int tng_transpose_bf16(const void* x, int64_t B, int64_t R, int64_t C, int64_t ld_x, void* y, int64_t ld_y,
                       void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused classifier-free guidance + scheduler update (one HBM pass).
 * Replaces: models.py:244-249 (chunk, uncond + g*(text-uncond)) and DDPMScheduler.step
 *           (scheduling_ddpm.py:290-344) / DDIMScheduler.step eta=0 (scheduling_ddim.py:292-354).
 * coef = float[10] {c_x0_sample, c_x0_model, c_prev_x0, c_prev_sample, c_noise, c_eps_sample, c_eps_model,
 *         c_prev_eps, clip (0 = off), c_x0_div}: fp32 scalars computed on the host with the reference's own fp32
 *         op order (device pointer, so a step can be replayed from a CUDA graph with updated coefficients).
 *   x0   = (c_x0_sample * sample + c_x0_model * v) / c_x0_div   (clamped to +-clip if clip > 0)
 *   eps  = c_eps_sample * sample + c_eps_model * v
 *   prev = c_prev_x0 * x0 + c_prev_sample * sample + c_prev_eps * eps + c_noise * noise
 * model_out: fp32 channels-last [(2)B, HW, C] (uncond half first when cfg); sample/noise/prev: fp32 NCHW
 * [B, C, HW] (the reference's latent layout); also writes next_in: the channels-last bf16 UNet input
 * [(2)B, HW, ld_in] for the next step (latents duplicated for the two CFG halves, hi/lo split optional).
 * Returns TNG_EINVAL, before any CUDA call, unless: the required pointers are non-NULL (sample, coef, and prev or
 * next_in); B, C, HW >= 1; ld_mo >= C when model_out is given; with next_in, split_off is 0 or >= C and
 * ld_in >= C + split_off. tng_dpm_step and tng_latent_blend make the same checks.
 */
int tng_sched_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                   const float* noise, const float* coef, float* prev, void* next_in, int64_t ld_in,
                   int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused classifier-free guidance + multistep DPM-Solver(++) update (one HBM pass).
 * Replaces: models.py:244-249 and DPMSolverMultistepScheduler.step (scheduling_dpmsolver_multistep.py:429-495:
 *           convert_model_output :243-281 and the order-1/2/3 updates :305-427).
 * coef = float[11] {c_a, c_b, c_d, c_s, c_0, c_1, c_2, 1/r0, 1/r1, r0/(r0+r1), 1/(r0+r1)}: fp32 scalars computed on
 *         the host with the reference's own fp32 op order, signs folded in (device pointer).
 *   v    = u + guidance * (t - u)  (cfg) or the model output itself
 *   m0   = (c_a * sample + c_b * v) / c_d                              written to the history slot m0
 *   order 1: x = c_s * sample - c_0 * m0
 *   order 2: x = (c_s * sample - c_0 * m0) + c_1 * D1,                D1 = (1/r0) * (m0 - m1)
 *   order 3: x = ((c_s * sample - c_0 * m0) + c_1 * D1) - c_2 * D2,   D1_0 = (1/r0) * (m0 - m1),
 *            D1_1 = (1/r1) * (m1 - m2), D1 = D1_0 + (r0/(r0+r1)) * (D1_0 - D1_1), D2 = (1/(r0+r1)) * (D1_0 - D1_1)
 * every product / sum is one round-to-nearest fp32 op (no fma), so x equals the reference's CPU fp32 result bit
 * for bit. model_out: fp32 channels-last [(2)B, HW, C] (uncond half first when cfg); sample, m0 / m1 / m2 (the
 * converted outputs of this, the previous and the one-before step; m1 is needed for order >= 2, m2 for order 3)
 * and prev: fp32 NCHW [B, C, HW]; prev may alias sample. The caller rotates the history slots. Also writes
 * next_in: the channels-last bf16 UNet input [(2)B, HW, ld_in] (duplicated for the CFG halves, hi/lo split at
 * split_off when > 0). TNG_EINVAL as tng_sched_step (required: model_out, sample, coef, m0, and prev or next_in), and
 * for an order outside 1-3 or a missing history slot.
 */
int tng_dpm_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                 const float* coef, int32_t order, float* m0, const float* m1, const float* m2, float* prev,
                 void* next_in, int64_t ld_in, int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused classifier-free guidance + multistep UniPC predictor-corrector update (one HBM pass).
 * Replaces: models.py:244-249 and UniPCMultistepScheduler.step (scheduling_unipc_multistep.py:490-572:
 *           convert_model_output :225-278, the UniC corrector :384-488 and the UniP predictor :279-382).
 * coef = float[18], fp32 scalars computed on the host with the reference's own fp32 op order (device pointer):
 *   [0..2]   {c_a, c_b, c_d}          conversion of the model output at this step's timestep t_i
 *   [3..10]  {c_x, c_m, c_b, r_0, r_1, rho_0, rho_1, rho_last}  corrector from s0 = t_{i-1} to t_i
 *   [11..17] {c_x, c_m, c_b, r_0, r_1, rho_0, rho_1}            predictor from s0 = t_i to t_{i+1}
 *   with c_x = sigma_t / sigma_s0, c_m = alpha_t * h_phi_1, c_b = alpha_t * B_h (alpha and sigma swapped when the
 *   solver predicts the noise), r_k = (lambda_{s_k} - lambda_s0) / h and rho the UniC / UniP weights.
 *   v    = u + guidance * (t - u)  (cfg) or the model output itself
 *   m    = (c_a * sample + c_b * v) / c_d                                  written to m_cur
 *   corrector (p = corrector_order >= 1; p = 0 skips it and x = sample):
 *     D_k  = (m_prev(k+1) - m_prev1) / r_k                                 k < p - 1
 *     corr = 0 (p = 1), rho_0 * D_0 (p = 2), fma(rho_1, D_1, rho_0 * D_0) (p = 3)
 *     x    = (c_x * last - c_m * m_prev1) - c_b * (corr + rho_last * (m - m_prev1))      written to last
 *   predictor (q = predictor_order):
 *     D_k  = (m_prev(k+1) - m) / r_k                                       k < q - 1
 *     res  = 0 (q = 1), rho_0 * D_0 (q = 2), fma(rho_1, D_1, rho_0 * D_0) (q = 3)
 *     prev = (c_x * x - c_m * m) - c_b * res
 * every other product / sum is one round-to-nearest fp32 op, so prev equals the reference's CPU fp32 result bit for
 * bit. model_out: fp32 channels-last [(2)B, HW, C] (uncond half first when cfg); sample, m_cur, m_prev1..3 (the
 * converted outputs of this step and of the 1..3 steps before), last (in: the corrected sample of the previous step;
 * out: this step's) and prev: fp32 NCHW [B, C, HW]. prev may alias sample; m_cur may alias no history slot it reads.
 * last may be NULL when p = 0. Also writes next_in: the channels-last bf16 UNet input [(2)B, HW, ld_in] (duplicated
 * for the CFG halves, hi/lo split at split_off when > 0). TNG_EINVAL as tng_sched_step (required: model_out, sample,
 * coef, m_cur, and prev or next_in), for p outside 0-3 or q outside 1-3, for a missing history slot among the
 * max(p, q - 1) it reads or one equal to m_cur, and for a missing last when p > 0.
 */
int tng_unipc_step(const float* model_out, int64_t ld_mo, int32_t cfg, float guidance, const float* sample,
                   const float* coef, int32_t corrector_order, int32_t predictor_order, float* m_cur,
                   const float* m_prev1, const float* m_prev2, const float* m_prev3, float* last, float* prev,
                   void* next_in, int64_t ld_in, int32_t split_off, int64_t B, int64_t C, int64_t HW, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Latent blend of text-guided editing / inpainting (one HBM pass), run after tng_sched_step / tng_dpm_step.
 * Replaces: the schedulers' add_noise (scheduling_ddpm.py:351-372; DDIM and DPM-Solver use the same formula) and the
 *           masking of StableDiffusionInpaintPipelineLegacy (pipeline_stable_diffusion_inpaint_legacy.py:692-709).
 * coef = float[2] {sqrt(alphas_cumprod[t]), sqrt(1 - alphas_cumprod[t])} computed on the host in fp32 (device pointer).
 *   p      = sqrt_a * x0 + sqrt_1ma * noise              (the noise term is dropped when noise == NULL)
 *   sample = p                                           (mask == NULL: add_noise)
 *   sample = p * m + sample * (1 - m)                    (mask: 1 keeps the noised input, 0 keeps sample)
 * every product / sum is one round-to-nearest fp32 op (no fma), so the result equals the fork's CPU fp32 ops bit for
 * bit; coef = {1, 0} with noise == NULL is the final blend x0 * m + sample * (1 - m). x0, noise, sample: fp32 NCHW
 * [B, C, HW]; sample is read only under a mask and may not alias x0 or noise. mask: fp32 [Bm, HW], entry b at
 * mask + b * mask_bstride (0 broadcasts one mask over the batch). Optionally also writes next_in: the channels-last
 * bf16 UNet input [(2)B, HW, ld_in] (duplicated for the CFG halves when cfg, hi/lo split at split_off when > 0), as
 * tng_sched_step packs it. TNG_EINVAL as tng_sched_step (required: x0, coef, sample), and for mask_bstride < 0.
 */
int tng_latent_blend(const float* x0, const float* noise, const float* mask, int64_t mask_bstride, const float* coef,
                     float* sample, void* next_in, int64_t ld_in, int32_t cfg, int32_t split_off, int64_t B, int64_t C,
                     int64_t HW, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Small exact-fp32 pieces.
 * tng_timestep_embedding: get_timestep_embedding (embeddings.py:22-62), flip_sin_to_cos / freq_shift configurable.
 * tng_linear_f32: y = act(x) @ W^T + b for tiny M (TimestepEmbedding, resnet time_emb_proj; embeddings.py:200-212,
 *                 resnet.py:572-573). pre_act is applied to x on load, post_act to y; each is TNG_ACT_NONE or
 *                 TNG_ACT_SILU (anything else is TNG_EINVAL).
 */
int tng_timestep_embedding(const float* t, int64_t n, int32_t dim, int32_t flip_sin_to_cos, float freq_shift,
                           float* out, void* stream);
int tng_linear_f32(const float* x, int64_t M, int64_t K, const float* w, const float* b, int64_t N,
                   int32_t pre_act, int32_t post_act, float* y, void* stream);

/* HiFi-GAN ConvTranspose1d overlap-add: y[b, l, co] = bias[co] + sum_{q,t: q*stride + t - pad = l} Y[b, q, t*Cout + co]
 * (audioldm/hifigan/models.py:124-135,153), Y being the tng_conv_gemm output [B, Lin, ktaps*Cout] fp32. */
int tng_convt_gather(const float* Y, int64_t B, int64_t Lin, int32_t ktaps, int64_t Cout, int32_t stride, int32_t pad,
                     int64_t Lout, const float* bias, float* y, void* stream);

/* Final waveform: tanh then the host-side `(x * 32768).astype(int16)` of hifigan/utilities.py:81
 * (C-style truncation toward zero; the +1.0 wrap-around of the reference is reproduced). */
int tng_tanh_to_i16(const float* x, int64_t n, int64_t ld_x, float* wave_f32, int16_t* wave_i16, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * TacotronSTFT mel front-end (SURVEY.md section 8(f).2): audioldm/audio/stft.py:52-83 (STFT.transform: reflect pad,
 * strided conv1d with the windowed Fourier basis, magnitude), :161-186 (mel_spectrogram), audio_processing.py:85-91
 * (log of the value clamped at 1e-5). The two contractions (basis, mel filter bank) run through tng_conv_gemm.
 * tng_stft_frames: y fp32 [B, T] -> reflect-padded by `pad` on both sides, split into bf16 hi / lo planes [B, ld]
 *   (ld >= T + 2 pad, zero beyond): frame f of batch b is the OVERLAPPING window [f hop, f hop + filter_length) of a plane,
 *   i.e. a tng_aview with s_w = hop — the conv1d needs no im2col buffer.
 * tng_stft_magnitude: F fp32 [rows, ldF] = (real | imag) halves of `bins` columns -> mag = sqrt(re^2 + im^2) as the bf16
 *   operand of the mel GEMM (hi at column b, lo at split_off + b; may be NULL), log_mag fp32 [rows, bins] =
 *   log(max(mag, floor)) (may be NULL), energy fp32 [rows] = ||mag||_2 (may be NULL).
 * tng_log_clamp: y = log(max(x, floor)). */
int tng_stft_frames(const float* y, int64_t B, int64_t T, int32_t pad, void* hi, void* lo, int64_t ld, void* stream);
int tng_stft_magnitude(const float* F, int64_t rows, int32_t bins, int64_t ldF, void* mag_op, int64_t ld_op,
                       int32_t split_off, float* log_mag, float* energy, float floor_v, void* stream);
int tng_log_clamp(const float* x, int64_t n, float floor_v, float* y, void* stream);

#ifdef __cplusplus
}
#endif
#endif
