/* kdiffusion_b200.h -- C ABI of libkdb200.so, the H100 (sm_90a) native library behind the
 * k_diffusion sampling hot path.
 *
 * The reference (crowsonkb/k-diffusion) is pure Python and has no FFI layer of its own
 * (SURVEY.md section 8b); these entry points are what a binding for the hot path would need.  Each
 * group cites the reference interface (file:line under the reference root) it replaces.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless named *_host; the library never takes ownership of
 *    caller memory and never allocates caller-visible memory (model-derived tables are owned by
 *    the KdbModel handle and released by kdb_model_destroy);
 *  - `stream` is a cudaStream_t passed as void*; every call is asynchronous and stream-ordered,
 *    legal inside CUDA-graph capture (no allocation / synchronisation inside forward or solver calls);
 *  - return value: 0 = ok, <0 = KDB_ERR_* (bad argument / unsupported), >0 = cudaError_t;
 *    kdb_last_error() returns a thread-local description of the last non-zero return;
 *  - latents are fp32 NCHW contiguous, like the reference's `x` (sample.py:59).
 */
#ifndef KDIFFUSION_B200_H
#define KDIFFUSION_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KDB_ABI_VERSION 28

#define KDB_ERR_BAD_ARG      (-1)
#define KDB_ERR_UNSUPPORTED  (-2)
#define KDB_ERR_MISSING_KEY  (-3)
#define KDB_ERR_BAD_SHAPE    (-4)
#define KDB_ERR_WORKSPACE    (-5)
#define KDB_ERR_NOT_FINAL    (-6)

int         kdb_abi_version(void);
const char* kdb_last_error(void);
/* Number of kernels this library has launched since load (process-wide, all streams). */
uint64_t    kdb_launch_count(void);
/* Per-kernel-family launch counters; fills names/counts up to `cap`, returns how many exist. */
int         kdb_launch_breakdown(const char** names, uint64_t* counts, int cap);

/* Per-launch device timing for bench.py's roofline leg (eager launches only, not capturable):
 * between begin and end every kernel this library launches is followed by an event on its stream;
 * kdb_profile_end synchronises, writes (family index into kdb_launch_breakdown names, milliseconds)
 * per launch into the host arrays and returns the number of launches seen. */
int kdb_profile_begin(int max_launches, void* stream);
int kdb_profile_end(int* families_host, float* ms_host, int cap);
/* Holds `stream` busy for `nanoseconds` (one spinning thread, bounded by the GPU's global timer, <= 2 s) so that the host can
 * enqueue the launches of a profiled region before the first of them runs: the kernels then execute back to back, as they do
 * under CUDA-graph replay, and the per-launch event intervals contain no host launch gaps.  Measurement aid only: it is not
 * counted by kdb_launch_count and never used on the product path. */
int kdb_profile_gate(int64_t nanoseconds, void* stream);

/* ------------------------------------------------------------------------------------------
 * Solver elementwise ops (HBM-bound, 128-bit vectorised).  n = number of fp32 elements.
 * Aliasing: `out` may alias any input of the same call.
 * ------------------------------------------------------------------------------------------ */

/* x_out = x + (x - den) * r  [+ noise * cn]
 * Euler step / Heun predictor with r = dt / sigma_hat  (sampling.py:129-134, 170-179: to_d + x + d*dt);
 * Euler-ancestral with r = (sigma_down - sigma_i)/sigma_i and cn = s_noise*sigma_up (sampling.py:149-154).
 * noise may be NULL (cn ignored). */
int kdb_solver_euler_step(const float* x, const float* den, const float* noise, float* x_out,
                          int64_t n, float r, float cn, void* stream);

/* x_out = x + (x - den1) * a1 + (x2 - den2) * a2
 * Heun corrector with a1 = dt/(2 sigma_hat), a2 = dt/(2 sigma_next)  (sampling.py:179-183). */
int kdb_solver_heun_correct(const float* x, const float* den1, const float* x2, const float* den2,
                            float* x_out, int64_t n, float a1, float a2, void* stream);

/* x_out = a * x - b * (k1 * den + k0 * old_den)      (old_den may be NULL when k0 == 0)
 * DPM-Solver++(2M): a = sigma_next/sigma, b = expm1(-h), k1 = 1 + 1/(2r), k0 = -1/(2r)
 * (sampling.py:598-605). */
int kdb_solver_dpmpp_2m_step(const float* x, const float* den, const float* old_den, float* x_out,
                             int64_t n, float a, float b, float k1, float k0, void* stream);

/* out = sum_i coef[i] * in[i],  1 <= n_in <= 6.  Generic N-ary axpby for the remaining
 * fixed-schedule samplers (SURVEY.md section 8f.1) and churn noise injection (sampling.py:168). */
int kdb_solver_lincomb(const float* const* in_host, const float* coef_host, int n_in, float* out,
                       int64_t n, void* stream);

/* out = uncond + (cond - uncond) * scale: classifier-free guidance combine of the two halves of a doubled batch
 * (train.py:333-344 make_cfg_model_fn), same operation order as the reference. */
int kdb_solver_cfg_combine(const float* uncond, const float* cond, float* out, int64_t n, float scale, void* stream);

/* partials[0] = sum_i ((x_low[i] - x_high[i]) / max(atol, rtol * max(|x_low[i]|, |x_prev[i]|)))^2 : the local error estimate of
 * the adaptive DPM-Solver (sampling.py:466-468; the caller takes sqrt(. / n)).  partials: device scratch of >= 512 floats;
 * deterministic (fixed grid, partial sums added in index order). */
#define KDB_DPM_ERROR_SCRATCH 512
int kdb_solver_dpm_error(const float* x_low, const float* x_high, const float* x_prev, int64_t n, float atol, float rtol,
                         float* partials, void* stream);

/* partials[0] = sum_i (err[i] / (atol + rtol * max(|y0[i]|, |y1[i]|)))^2 : the error ratio of an embedded Runge-Kutta step
 * (the dopri5 integration behind log_likelihood, sampling.py:280-301; the caller takes sqrt(. / n)).  Same scratch and
 * determinism contract as kdb_solver_dpm_error. */
int kdb_solver_rk_error(const float* err, const float* y0, const float* y1, int64_t n, float atol, float rtol,
                        float* partials, void* stream);

/* out[b,...] = (x[b,...] - den[b,...]) / sigma[b]      (sampling.py:46-48 to_d; sigma is [B]) */
int kdb_solver_to_d(const float* x, const float* den, const float* sigma, float* out,
                    int batch, int64_t per_sample, void* stream);

/* Karras preconditioner pieces for an opaque inner model (layers.py:70-74,88-90); sigma is [B].
 *   kdb_precond_scale_in : out[b,...] = x[b,...] * c_in(sigma[b])
 *   kdb_precond_combine  : out[b,...] = f[b,...] * c_out(sigma[b]) + x[b,...] * c_skip(sigma[b]) */
int kdb_precond_scale_in(const float* x, const float* sigma, float sigma_data, float* out,
                         int batch, int64_t per_sample, void* stream);
int kdb_precond_combine(const float* f, const float* x, const float* sigma, float sigma_data, float* out,
                        int batch, int64_t per_sample, void* stream);

/* Training losses with the Karras preconditioner, scales == 1 (layers.py:76-86 Denoiser.loss, :107-111 SimpleLossDenoiser.loss); x (the
 * clean input), noise [B, ...], sigma [B], sigma_data > 0, per_sample elements per image.
 *   kdb_loss_noised_input: out = (x + noise * sigma) * c_in(sigma), the inner model's input
 *   kdb_denoiser_loss:     f = the inner model's output on it.  KDB_LOSS_DENOISER: loss[b] = mean((f - target)^2) * weight[b],
 *                          target = (x - c_skip * (x + noise sigma)) / c_out.  KDB_LOSS_SIMPLE (weight unused): loss[b] = mean((eps - noise)^2),
 *                          eps = ((x + noise sigma) - (f c_out + (x + noise sigma) c_skip)) / sigma.  cotangent (or NULL) receives d loss[b] / d f.
 * One CTA per image, a fixed-order sum: two calls give the same bits. */
#define KDB_LOSS_DENOISER 0
#define KDB_LOSS_SIMPLE   1
int kdb_loss_noised_input(const float* x, const float* noise, const float* sigma, float sigma_data, float* out,
                          int batch, int64_t per_sample, void* stream);
int kdb_denoiser_loss(int kind, const float* x, const float* noise, const float* sigma, const float* weight, float sigma_data,
                      const float* f, float* loss, float* cotangent, int batch, int64_t per_sample, void* stream);

/* The training loss of a model with a learned variance (layers.py:93-101 DenoiserWithVariance.loss), with the arguments of
 * kdb_denoiser_loss and logvar [B], the model's per-image log-variance (kdb_unet_forward_variance): with m = mean((f - target)^2),
 * loss[b] = (m exp(-logvar[b]) + logvar[b]) / 2; cotangent (or NULL) receives d loss[b] / d f = (f - target) exp(-logvar[b]) / per_sample,
 * dlogvar (or NULL) d loss[b] / d logvar[b] = (1 - m exp(-logvar[b])) / 2.  m, loss and dlogvar are formed in double and rounded once,
 * since 1 - m exp(-logvar) cancels as the variance fits.  One CTA per image, a fixed-order sum: two calls give the same bits. */
int kdb_variance_loss(const float* x, const float* noise, const float* sigma, float sigma_data, const float* f, const float* logvar, float* loss,
                      float* cotangent, float* dlogvar, int batch, int64_t per_sample, void* stream);

/* The per-evaluation math of the external model wrappers (external.py:9-38, 87-177: VDenoiser, DiscreteEpsDDPMDenoiser,
 * OpenAIDenoiser, CompVisDenoiser, DiscreteVDDPMDenoiser, CompVisVDenoiser); sigma is [B] fp32.  Every product and sum is
 * rounded on its own (no FMA contraction), in the order the reference's torch expressions evaluate, so on the same GPU the
 * result equals the reference's fp32 expression bit for bit.  With s2 = sigma^2 + sigma_data^2:
 *   kdb_external_scale_in : out[b,...] = x[b,...] * c_in,   c_in = 1 / sqrt(s2)
 *   kdb_external_combine  : kind KDB_EXTERNAL_EPS  out[b,...] = x[b,...] + f[b,...] * (-sigma[b])
 *                           kind KDB_EXTERNAL_V    out[b,...] = f[b,...] * c_out + x[b,...] * c_skip,
 *                                                  c_out = -sigma sigma_data / sqrt(s2), c_skip = (1 / s2) sigma_data^2
 * `f` is the inner model's output as it stands: dtype KDB_DTYPE_F32 / F16 / BF16 (converted to fp32 exactly), each sample
 * a contiguous run of per_sample elements, sample b starting at f + b * f_batch_stride elements (so the eps half of a
 * learned-variance output, output[:, :C], is read in place).  Either of `f` and `x` may be NULL, which drops its term:
 * the derivatives (g_eps = -sigma u, g_v = c_out u, g_x = c_skip u and the tangents) run on the same kernel. */
#define KDB_EXTERNAL_EPS 0
#define KDB_EXTERNAL_V   1
#define KDB_DTYPE_F32    0
#define KDB_DTYPE_F16    1
#define KDB_DTYPE_BF16   2
int kdb_external_scale_in(const float* x, const float* sigma, float sigma_data, float* out, int batch, int64_t per_sample,
                          void* stream);
int kdb_external_combine(int kind, const void* f, int f_dtype, int64_t f_batch_stride, const float* x, const float* sigma,
                         float sigma_data, float* out, int batch, int64_t per_sample, void* stream);

/* Counter-based standard-normal fill (Philox4x32-10 + Box-Muller): element i of sample b gets the
 * (seed[b], stream_id, i) variate, so results do not depend on how a batch is sharded across GPUs.
 * Replaces torch.randn_like in default_noise_sampler (sampling.py:61-62).  seeds is a device int64 [B]. */
int kdb_noise_normal(float* out, const int64_t* seeds, uint64_t stream_id, int batch, int64_t per_sample,
                     void* stream);

/* Virtual Brownian bridge increment W(t1) - W(t0), normalised by sqrt(|t1 - t0|), per sample.
 * Replaces BatchedBrownianTree / BrownianTreeNoiseSampler (sampling.py:65-114): dyadic Brownian-bridge
 * tree on [t_min, t_max] of `depth` levels evaluated from (seed[b], node, element) counters.
 * Parity with torchsde is UNPINNED (torchsde absent).  The values are pinned instead: oracle/counter_noise.py restates the counter
 * stream in float64 and tests/test_gpu_noise.py holds this kernel to it element by element.
 * t0 and t1 are clamped to [t_min, t_max], but the norm is the UNCLAMPED sqrt(|t1 - t0|): a call reaching outside the interval
 * returns increments of variance |clamped span| / |t1 - t0| < 1.  The samplers never make such a call. */
int kdb_noise_brownian(float* out, const int64_t* seeds, int batch, int64_t per_sample,
                       double t_min, double t_max, double t0, double t1, int depth, void* stream);

/* ------------------------------------------------------------------------------------------
 * image_transformer_v2 denoiser engine (models/image_transformer_v2.py:667-762, layers.py:45-90), which also runs
 * image_transformer_v1 (models/image_transformer_v1.py:280-344) as a one-level model with global attention
 * ------------------------------------------------------------------------------------------ */

#define KDB_MAX_LEVELS 8

enum { KDB_ATTN_NONE = 0, KDB_ATTN_GLOBAL = 1, KDB_ATTN_NEIGHBORHOOD = 2, KDB_ATTN_SHIFTED_WINDOW = 3 };
/* arithmetic of the token stream / GEMM operands.  KDB_PREC_TF32 and KDB_PREC_FP16 (the image_v1 U-Net only; every kdb_model_* entry
 * point returns KDB_ERR_UNSUPPORTED for them): convolution and attention operands rounded to tf32 / fp16, fp32 accumulation, fp32
 * activations and outputs.  fp16 rounding is to nearest even without saturation: an operand of magnitude >= 65520 becomes +-inf. */
enum { KDB_PREC_FP32 = 0, KDB_PREC_BF16 = 1, KDB_PREC_TF32 = 2, KDB_PREC_FP16 = 3 };
/* KdbModelConfig.family.  KDB_FAMILY_ITV1: image_transformer_v1 with n_levels 1, width = depth's d_model, d_ff, attn_type
 * KDB_ATTN_GLOBAL, d_head 64, mapping_width = d_model, mapping_depth 2, mapping_d_ff = d_ff, mapping_cond_dim 0.  Its keys are v1's own
 * ("blocks.<i>.self_attn.qk_norm.scale", "in_proj.weight", ...); kdb_model_finalize derives the engine's tables from them: qkv_proj
 * with the q and k rows of each head permuted (new column j <- 2j, j + 32 <- 2j + 1), the cosine-sim scale exp(min(qk_norm.scale,
 * ln 100)) with eps 64e-6 (QKNorm + SDPA's 1/sqrt(d_head)), the RoPE frequencies exp(freqs_h) | exp(freqs_w) over all 64 columns, and
 * in_proj's columns / out_proj's rows reordered from v1's patch feature order (c i j) to the engine's (i j c).  Positions follow the
 * image's aspect ratio W / H (v1's pixel_aspect_ratio = patch_h / patch_w).  The ".qkv" debug tap then holds q and k in the permuted
 * column order. */
enum { KDB_FAMILY_ITV2 = 0, KDB_FAMILY_ITV1 = 1 };

typedef struct KdbModelConfig {
  int32_t n_levels;                       /* len(levels); last level is the mid level       (:682-699) */
  int32_t in_channels, out_channels;
  int32_t patch_h, patch_w;               /* TokenMerge patch_in / TokenSplitWithoutSkip    (:672,705) */
  int32_t mapping_width, mapping_depth, mapping_d_ff;   /* MappingSpec                      (:657-662) */
  int32_t num_classes;                    /* rows of class_emb (0 = unconditional)           (:678)     */
  int32_t mapping_cond_dim;               /* 0 = none                                        (:679)     */
  int32_t width[KDB_MAX_LEVELS];          /* LevelSpec                                       (:648-654) */
  int32_t depth[KDB_MAX_LEVELS];
  int32_t d_ff[KDB_MAX_LEVELS];
  int32_t attn_type[KDB_MAX_LEVELS];      /* KDB_ATTN_*                                                 */
  int32_t d_head[KDB_MAX_LEVELS];
  int32_t attn_param[KDB_MAX_LEVELS];     /* kernel_size (neighborhood) / window_size (shifted window)  */
  int32_t family;                         /* KDB_FAMILY_*                                               */
} KdbModelConfig;

typedef struct KdbModel KdbModel;

int  kdb_model_create(const KdbModelConfig* cfg, KdbModel** out);
void kdb_model_destroy(KdbModel* m);

/* Bind one state-dict entry (fp32, contiguous, device) by its reference key name, e.g.
 * "down_levels.0.1.self_attn.qkv_proj.weight" (key list: SURVEY.md section 8b), or for KDB_FAMILY_ITV1
 * "blocks.3.self_attn.pos_emb.freqs_h".  The pointer is
 * borrowed: it must stay valid until the next kdb_model_finalize or destroy.  Replaces
 * nn.Module.load_state_dict for the engine (sample.py:44). */
int kdb_model_set_tensor(KdbModel* m, const char* key, const float* data, const int64_t* shape, int ndim);

/* Validate that every required key is bound with the right shape and (re)build derived device
 * tables (bf16 / reordered weight copies, concatenated AdaRMSNorm projection, RoPE tables).
 * Must be called after weights change and before forward.  Synchronises `stream`. */
int kdb_model_finalize(KdbModel* m, void* stream);

/* Floats per row of the conditioning table produced by kdb_model_conditioning. */
int64_t kdb_model_cond_stride(const KdbModel* m);

/* Mapping network + every AdaRMSNorm projection for `rows` (sigma, aug, class, mapping_cond) tuples
 * (image_transformer_v2.py:734-740 and :166 for each block).  cond_out is [rows, cond_stride] fp32.
 * aug_cond [rows,9] / class_cond [rows] int64 / mapping_cond [rows,dim] may be NULL where the
 * reference allows None.  Because the sigma schedule is known before the solver loop starts, a
 * sampler calls this ONCE for all steps (rows = n_model_evals * batch). */
int kdb_model_conditioning(KdbModel* m, int rows, const float* sigma, const float* aug_cond,
                           const int64_t* class_cond, const float* mapping_cond, float* cond_out, void* stream);

size_t kdb_model_workspace_bytes(const KdbModel* m, int precision, int batch, int height, int width);

/* One denoiser evaluation on x [B, C_in, H, W] -> out [B, C_out, H, W].
 *   sigma_data > 0 : Karras-preconditioned  D(x, sigma) = c_skip x + c_out F(c_in x, sigma)
 *                    (layers.py:88-90; requires C_in == C_out); sigma is [B];
 *   sigma_data <= 0: the raw inner model F(x, sigma) (image_transformer_v2.py:721-762).
 * cond holds rows from kdb_model_conditioning for the same sigma/conditioning; sample b reads the
 * row at cond + b * cond_batch_stride (floats): cond_stride for per-sample rows, 0 when the whole
 * batch shares one (sigma, conditioning) tuple -- the usual case inside a sampler.  With a shared row (and the bf16
 * precision) every AdaRMSNorm is fused into the neighbouring GEMMs: the channel scales are folded into per-evaluation
 * copies of the qkv / up_proj weights and 1/rms comes from row statistics the producing GEMM leaves in the workspace.
 * All launches are stream-ordered on `stream` (several with programmatic dependent launch, i.e. a kernel's prologue may
 * overlap the tail of its predecessor on the same stream); nothing is allocated or synchronised, so the call can be
 * captured into a CUDA graph once the position tables of this token grid exist (first call outside capture). */
int kdb_model_forward(KdbModel* m, int precision, int batch, int height, int width,
                      const float* x, const float* sigma, float sigma_data,
                      const float* cond, int64_t cond_batch_stride, float* out,
                      void* workspace, size_t workspace_bytes, void* stream);

/* Forward-mode derivative (JVP) of the same evaluation along v [B, C_in, H, W]: out = D(x, sigma) as kdb_model_forward computes it at
 * KDB_PREC_FP32 (bit for bit), out_tangent = J_D(x) v = c_skip v + c_out J_F(c_in x) c_in v (sigma_data > 0) or J_F(x) v (sigma_data <= 0).
 * The derivative is taken with respect to x only (sigma and the conditioning are held fixed).  fp32 only: any other precision returns
 * KDB_ERR_UNSUPPORTED.  The tangent rides through the engine as images [B, 2B) of every token buffer, so the workspace must hold
 * kdb_model_workspace_bytes(m, KDB_PREC_FP32, 2 * batch, height, width) bytes.  cond / cond_batch_stride as for kdb_model_forward:
 * tangent image b uses the conditioning row of image b.  Armed debug taps receive the primal rows followed by the tangent rows.  Same
 * stream, allocation and CUDA-graph rules as kdb_model_forward. */
int kdb_model_forward_jvp(KdbModel* m, int precision, int batch, int height, int width,
                          const float* x, const float* v, const float* sigma, float sigma_data,
                          const float* cond, int64_t cond_batch_stride, float* out, float* out_tangent,
                          void* workspace, size_t workspace_bytes, void* stream);

/* Reverse-mode derivative (VJP) of the same evaluation for a cotangent u [B, C_out, H, W]: out = D(x, sigma) as kdb_model_forward computes it
 * at KDB_PREC_FP32 (bit for bit), grad_x = u^T J_D(x) = c_skip u + c_in J_F(c_in x)^T (c_out u) (sigma_data > 0) or J_F(x)^T u
 * (sigma_data <= 0), shape of x.  The derivative is taken with respect to x only (sigma and the conditioning are held fixed).  fp32 only:
 * any other precision returns KDB_ERR_UNSUPPORTED.  The forward keeps the fp32 residual stream entering every attention half, every
 * feed-forward half and out_norm on a tape; the backward walks the layers in reverse, recomputes each half's activations from its tape
 * entry with the forward's own launches and runs the backward kernels.  The workspace holds one fp32 forward workspace of `batch` images,
 * the tape and the gradient buffers: kdb_model_vjp_workspace_bytes returns its size in bytes (or a negative KDB_ERR_* for a NULL model
 * or a non-positive size; kdb_model_workspace_bytes is unchanged), a shorter one returns KDB_ERR_WORKSPACE.  cond / cond_batch_stride
 * as for kdb_model_forward.  No atomics: two calls on the same inputs return the same bits.  Same stream, allocation and CUDA-graph
 * rules as kdb_model_forward. */
int64_t kdb_model_vjp_workspace_bytes(const KdbModel* m, int batch, int height, int width);
int kdb_model_forward_vjp(KdbModel* m, int precision, int batch, int height, int width,
                          const float* x, const float* sigma, float sigma_data,
                          const float* cond, int64_t cond_batch_stride,
                          const float* cotangent, float* out, float* grad_x,
                          void* workspace, size_t workspace_bytes, void* stream);

/* Parameter gradients (training) of an image_transformer_v2 model.  kdb_model_set_grad binds a gradient buffer [shape] fp32 on the device to
 * the state-dict key of a parameter, as kdb_model_set_tensor binds weights (data == NULL unbinds the key); binding needs no finalize.
 * kdb_model_forward_train runs the raw model F (sigma_data 0) forward at the training precision `precision` (below; at KDB_PREC_FP32 bit for
 * bit as kdb_model_forward), takes the cotangent u [B, C_out, H, W] on out = F(x, sigma) and OVERWRITES every bound gradient with u^T
 * dF/dparam summed over the batch; grad_x (shape of x, or NULL) receives u^T dF/dx.  Unbound parameters are skipped.  The walk is that of
 * kdb_model_forward_vjp with the weight gradients added, then the AdaRMSNorm projections and the mapping network (which is why the raw
 * conditioning inputs are passed: sigma [B], aug_cond [B, 9] or NULL, class_cond [B] int64 when num_classes > 0, mapping_cond [B,
 * mapping_cond_dim] when mapping_cond_dim > 0).  cond holds one conditioning row per image (kdb_model_conditioning of those inputs;
 * cond_batch_stride == kdb_model_cond_stride).  Bind the weights first: kdb_model_set_grad returns KDB_ERR_MISSING_KEY for a key that is no
 * tensor set on the model, KDB_ERR_BAD_SHAPE for a shape other than that tensor's, and KDB_ERR_BAD_ARG for the buffers time_emb.weight,
 * aug_emb.weight and *.pos_emb.freqs, which take no gradient; kdb_model_forward_train repeats these checks for every bound key (the weights
 * may have been rebound since) and returns the same codes.  The workspace is kdb_model_train_workspace_bytes(m, batch, height, width) bytes
 * (the finalized model's size; negative KDB_ERR_* on bad arguments).  No atomics: every sum over tokens or images runs in an order fixed by
 * the shapes, so two calls give the same bits.  Same stream and allocation rules as kdb_model_forward. */
int     kdb_model_set_grad(KdbModel* m, const char* key, float* data, const int64_t* shape, int ndim);
int64_t kdb_model_train_workspace_bytes(const KdbModel* m, int batch, int height, int width);
int     kdb_model_forward_train(KdbModel* m, int precision, int batch, int height, int width,
                                const float* x, const float* sigma, const float* aug_cond, const int64_t* class_cond,
                                const float* mapping_cond, const float* cond, int64_t cond_batch_stride,
                                const float* cotangent, float* out, float* grad_x,
                                void* workspace, size_t workspace_bytes, void* stream);

/* The training precision, `precision` of kdb_model_forward_train and kdb_model_train_forward: KDB_PREC_FP32 (the exact path above) or
 * KDB_PREC_TF32.  Any other value returns KDB_ERR_UNSUPPORTED, as does any value on an image_transformer_v1 handle, and KDB_PREC_TF32 when a
 * level's width or d_ff is not a multiple of 4; these checks come before the finalize check.  At KDB_PREC_TF32 each of the token-stream
 * Linears (qkv_proj, out_proj, up_proj, down_proj, merges.*.proj, splits.*.proj) runs, in the forward, in the input gradients and in the weight
 * gradients, on the tensor cores with tf32 operands (activations and output gradients truncated to tf32, weights rounded to the nearest tf32,
 * ties away from zero) and fp32 accumulation; patch_in, patch_out, every norm, cosine-sim + RoPE, GEGLU, the attention, the mapping network and
 * the conditioning stay exact fp32.  Still deterministic, no atomics.  The first KDB_PREC_TF32 call after a kdb_model_finalize builds two
 * copies of every token-stream weight, one rounded and its transpose rounded alike, in memory the handle keeps until kdb_model_destroy; that
 * call must run outside CUDA-graph capture (KDB_ERR_UNSUPPORTED otherwise).  The workspace of kdb_model_train_workspace_bytes is the same at
 * both precisions.
 * kdb_model_train_forward: the forward of kdb_model_forward_train without the reverse walk: F(x), or with sigma_data > 0 the
 * Karras-preconditioned D, bit for bit as kdb_model_forward_train's out at the same precision (KDB_PREC_FP32: as kdb_model_forward at
 * KDB_PREC_FP32).  Arguments, workspace (kdb_model_workspace_bytes at KDB_PREC_FP32) and rules as for kdb_model_forward. */
int kdb_model_train_forward(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                            const float* cond, int64_t cond_batch_stride, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Debug/parity tap: arm a copy of one intermediate of the NEXT forward into `out` (fp32, device).
 * name: "patch_in", "L<l>.down", "L<l>.merge", "mid", "L<l>.split", "L<l>.up", "layer<k>.xn1",
 * "layer<k>.qkv", "layer<k>.ao", "layer<k>.attn", "layer<k>.ff" (k = execution order).
 * After the forward, kdb_model_tap_count returns the number of floats written (0 = name never hit,
 * <0 = capacity too small).  The tap disarms itself after one forward. */
int     kdb_model_debug_tap(KdbModel* m, const char* name, float* out, int64_t capacity);
int64_t kdb_model_tap_count(const KdbModel* m);

/* ------------------------------------------------------------------------------------------
 * image_v1 U-Net denoiser engine, exact fp32 path (models/image_v1.py, layers.py:116-313, augmentation.py:92-104)
 * ------------------------------------------------------------------------------------------
 * A separate handle with the same life cycle as KdbModel: create, bind every state-dict entry, finalize, then fill a
 * conditioning table once per sampler call and run forwards.  Activations are token-major [B, H, W, C] fp32 inside the
 * workspace.  Every entry point returns a negative KDB_ERR_* for a NULL handle before any CUDA call. */

typedef struct KdbUNetConfig {
  int32_t n_levels;                       /* len(depths)                                               (image_v1.py:107-115) */
  int32_t in_channels;                    /* input_channels = c_in                                                           */
  int32_t patch_size;                     /* pixel_unshuffle / pixel_shuffle factor                    (:146-154)            */
  int32_t mapping_out;                    /* feats_in of the mapping net and every AdaGN mapper        (:97-100)             */
  int32_t mapping_cond_dim;               /* in-features of the mapping_cond Linear, 0 = none; 9 more with the augment wrapper */
  int32_t augment_wrapper;                /* 1: KarrasAugmentWrapper, mapping_cond = cat(aug_cond or zeros(9), mapping_cond)  */
  int32_t skip_stages;
  int32_t has_variance;                   /* proj_out has one extra (dropped) output channel           (:151-152)            */
  int32_t depth[KDB_MAX_LEVELS];          /* ResConvBlocks per DBlock / UBlock                                               */
  int32_t channels[KDB_MAX_LEVELS];       /* multiples of 4                                                                  */
  int32_t self_attn[KDB_MAX_LEVELS];      /* self_attn_depths                                                                */
} KdbUNetConfig;

typedef struct KdbUNet KdbUNet;

int kdb_unet_create(const KdbUNetConfig* cfg, KdbUNet** out);
int kdb_unet_destroy(KdbUNet* m);

/* Bind one state-dict entry of ImageDenoiserModelV1 (fp32, contiguous, device) by its reference key name, e.g.
 * "u_net.d_blocks.1.2.main.2.weight"; a KarrasAugmentWrapper's "inner_model." prefix is not part of the name.  Borrowed until
 * the next finalize or destroy. */
int kdb_unet_set_tensor(KdbUNet* m, const char* key, const float* data, const int64_t* shape, int ndim);

/* Validate every required key and build the derived tables: tap-major convolution weights, qkv_proj with 1/sqrt(d_head) folded
 * into its q rows and bias, the concatenated AdaGN mappers.  Synchronises `stream`. */
int kdb_unet_finalize(KdbUNet* m, void* stream);

/* Floats per conditioning row: the (weight, bias) pair of every AdaGN in execution order, then the mapping net's output. */
int64_t kdb_unet_cond_stride(const KdbUNet* m);

/* Fourier features of log(sigma)/4, the mapping_cond Linear, the mapping net and every AdaGN mapper for `rows` tuples
 * (image_v1.py:136-139, layers.py:173).  aug_cond [rows, 9] (augment wrapper only; NULL = zeros) and mapping_cond
 * [rows, mapping_cond_dim minus the wrapper's 9] may be NULL where the reference allows None. */
int kdb_unet_conditioning(KdbUNet* m, int rows, const float* sigma, const float* aug_cond, const float* mapping_cond, float* cond_out,
                          void* stream);

/* Workspace of one forward in bytes, the same at KDB_PREC_FP32, KDB_PREC_TF32 and KDB_PREC_FP16; KDB_ERR_UNSUPPORTED for any other
 * precision. */
int64_t kdb_unet_workspace_bytes(const KdbUNet* m, int precision, int batch, int height, int width);

/* One evaluation on x [B, in_channels, H, W] -> out of the same shape, as kdb_model_forward: sigma_data > 0 gives the
 * Karras-preconditioned denoiser, sigma_data <= 0 the raw inner model; cond rows with cond_batch_stride (0 = one shared row).
 * KDB_PREC_FP32: every kernel in fp32.  KDB_PREC_TF32: every convolution (the ResConvBlock 3x3 convs and 1x1 skip, qkv_proj and
 * out_proj) on the tensor cores (kdb_unet_conv_tf32) with weights rounded to tf32 by finalize, and self-attention of d_head 64 on the
 * tensor cores (kdb_attention at KDB_PREC_TF32; other head sizes keep the fp32 kernel); AdaGN, resampling, patch in / out and the
 * conditioning stay fp32.  KDB_PREC_FP16: the same with fp16 operands (kdb_unet_conv_fp16 on fp16 weight copies made by finalize,
 * kdb_attention at KDB_PREC_FP16).  Any other precision: KDB_ERR_UNSUPPORTED.  Every level but the innermost needs an even grid and every
 * level at least 2x2.  Allocates nothing and synchronises nothing, so it can be captured into a CUDA graph; a workspace shorter
 * than kdb_unet_workspace_bytes returns KDB_ERR_WORKSPACE.  Deterministic (no atomics). */
int kdb_unet_forward(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                     const float* cond, int64_t cond_batch_stride, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* kdb_unet_forward of a has_variance model (KDB_ERR_BAD_ARG for any other), whose `out` it writes bit for bit, plus the learned log-variance
 * logvar [B] (image_v1.py:151-152, return_variance=True): proj_out's variance channel averaged over the (H/p) x (W/p) token grid, computed
 * in fp32 from the features the forward's proj_out reads at every precision.  Same workspace. */
int kdb_unet_forward_variance(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                              const float* cond, int64_t cond_batch_stride, float* out, float* logvar, void* workspace, size_t workspace_bytes,
                              void* stream);

/* Debug/parity tap of the NEXT forward, token-major [B, h, w, C] fp32: "patch_in", "d<l>.down", "d<l>.<i>", "u<l>.<i>",
 * "u<l>.up" -- level l, i the module index inside the reference's DBlock (1..) / UBlock (0..), i.e. the output of that
 * ResConvBlock or SelfAttention2d.  kdb_unet_tap_count: floats written (0 = not hit, < 0 = capacity too small). */
int     kdb_unet_debug_tap(KdbUNet* m, const char* name, float* out, int64_t capacity);
int64_t kdb_unet_tap_count(const KdbUNet* m);

/* Parameter gradients (training) of the U-Net, exact fp32, as kdb_model_set_grad / kdb_model_forward_train do for image_transformer_v2.
 * kdb_unet_set_grad binds a gradient buffer [shape] fp32 on the device to the state-dict key of a parameter (data == NULL unbinds it):
 * KDB_ERR_MISSING_KEY for a key that is no tensor set on the model, KDB_ERR_BAD_SHAPE for a shape other than that tensor's, KDB_ERR_BAD_ARG
 * for the buffers timestep_embed.weight and *.kernel (the resampling filters), which take no gradient, and for the parameters of the DBlocks
 * and UBlocks of the levels below skip_stages, which the forward never runs.
 * kdb_unet_forward_train runs the raw model F (sigma_data 0) forward, bit for bit as kdb_unet_forward at KDB_PREC_FP32, takes the cotangent
 * u [B, in_channels, H, W] on out = F(x, sigma) and OVERWRITES every bound gradient with u^T dF/dparam summed over the batch (proj_out's
 * variance row of a has_variance model: exactly 0); unbound parameters are skipped.  sigma [B], aug_cond [B, 9] or NULL and mapping_cond are
 * the raw conditioning inputs as for kdb_unet_conditioning, cond one conditioning row per image made from them (cond_batch_stride ==
 * kdb_unet_cond_stride).  precision must be KDB_PREC_FP32 (KDB_ERR_UNSUPPORTED otherwise).  The bound keys are checked again, with
 * kdb_unet_set_grad's codes.  The first call after a kdb_unet_finalize builds the input-gradient copy of every convolution weight (taps
 * reversed, channels swapped) in memory the handle keeps until kdb_unet_destroy; that call must run outside CUDA-graph capture
 * (KDB_ERR_UNSUPPORTED otherwise).  The workspace is kdb_unet_train_workspace_bytes(m, batch, height, width) bytes (finalized model; negative
 * KDB_ERR_* on bad arguments); it holds the tape of every module's output.  No atomics: every sum runs in an order fixed by the shapes, so
 * two calls give the same bits. */
int     kdb_unet_set_grad(KdbUNet* m, const char* key, float* data, const int64_t* shape, int ndim);
int64_t kdb_unet_train_workspace_bytes(const KdbUNet* m, int batch, int height, int width);
int     kdb_unet_forward_train(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma,
                               const float* aug_cond, const float* mapping_cond, const float* cond, int64_t cond_batch_stride,
                               const float* cotangent, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* kdb_unet_forward_train of a has_variance model (KDB_ERR_BAD_ARG for any other) with the cotangent dlogvar [B] of its log-variance as
 * well: every bound gradient = u^T dF/dparam + dlogvar^T dlogvar/dparam, which reaches proj_out's variance row and, through it, every
 * parameter upstream.  Same arguments, checks, workspace and precision otherwise. */
int     kdb_unet_forward_train_variance(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma,
                                        const float* aug_cond, const float* mapping_cond, const float* cond, int64_t cond_batch_stride,
                                        const float* cotangent, const float* dlogvar, float* out, void* workspace, size_t workspace_bytes,
                                        void* stream);

/* ------------------------------------------------------------------------------------------
 * Stand-alone kernels exposed for unit tests / profiling (same code the engine launches)
 * ------------------------------------------------------------------------------------------ */

/* The parameter-gradient reductions of kdb_model_forward_train (the launches it makes).  No atomics: every sum is split into chunks fixed
 * by the shapes alone, each chunk summed in row order into scratch (caller scratch of 2^22 floats) and the partials summed in chunk order,
 * so two calls on the same inputs give the same bits.  Every element of the output is written.  Arguments are checked before any launch.
 *
 * kdb_wgrad: the weight gradient of a Linear, dw[n, k] = sum over rows r < m of dy[r, n] x[r, k].  KDB_PREC_FP32: fp32 fmaf products and
 * sums; KDB_PREC_TF32: dy and x truncated to tf32 (the low 13 mantissa bits cleared), products accumulated in fp32 on the tensor cores
 * (mma.sync); other precisions KDB_ERR_UNSUPPORTED.  dy rows ldy floats apart (>= n) in both modes, x rows ldx (>= k); with merge_hc,
 * merge_wc > 0, x is instead read in place as the TokenMerge 2x2 gather of contiguous fine tokens [m / (merge_hc merge_wc), 2 merge_hc,
 * 2 merge_wc, k / 4] (ldx unused; m a multiple of merge_hc merge_wc, k of 4). */
int kdb_wgrad(int precision, const float* dy, int64_t ldy, const float* x, int64_t ldx, float* dw, int64_t m, int n, int k, int merge_hc,
              int merge_wc, float* scratch, void* stream);
/* patch_in's weight gradient, fp32: dw [n, patch_h patch_w channels] = sum over the tokens t of dtok[t, n] (contiguous, [batch T, n]) times
 * the patch row of t in the NCHW image x [batch, channels, height, width], read in place, columns in the order (ph pw c). */
int kdb_wgrad_patch_in(const float* dtok, const float* x, float* dw, int batch, int channels, int height, int width, int patch_h, int patch_w,
                       int n, float* scratch, void* stream);
/* patch_out's weight gradient, fp32: dw [patch_h patch_w channels, c0] = sum over the tokens t of the patch row of t in u [batch, channels,
 * height, width] times out_norm's output tokens[t, :] * (scale * rstd[t]) (tokens [batch T, c0], scale [c0], rstd [batch T]). */
int kdb_wgrad_patch_out(const float* u, const float* tokens, const float* scale, const float* rstd, float* dw, int batch, int channels,
                        int height, int width, int patch_h, int patch_w, int c0, float* scratch, void* stream);
/* An RMSNorm channel scale's gradient per image: out[b ldo + j] = sum over the rows r of image b of dy[r, j] x[r, j] rstd_r, rstd_r =
 * rsqrt(mean_j x[r, j]^2 + 1e-6) recomputed in fp32; x rows ldx floats apart, dy rows ldy (both >= c); rows a multiple of rows_per_image
 * (rows_per_image == rows: one sum over all rows, ldo unused; else ldo >= c).  KDB_ERR_BAD_SHAPE when (rows / rows_per_image) times
 * ceil(rows_per_image / 64) times c exceeds 2^22. */
int kdb_norm_scale_grad(const float* x, int64_t ldx, const float* dy, int64_t ldy, float* out, int64_t ldo, int64_t rows_per_image,
                        int64_t rows, int c, float* scratch, void* stream);
/* Column sums: out[j] = sum over r < rows of p[r, j], p contiguous [rows, c].  KDB_ERR_BAD_SHAPE when ceil(rows / 256) c exceeds 2^22. */
int kdb_colsum(const float* p, int64_t rows, int c, float* out, float* scratch, void* stream);
/* TokenSplit's fac gradient: out[0] = sum of (y - skip) dup over the elements of skip and dup [batch, height, width, c], y [batch, height / 2,
 * width / 2, 4 c] the split projection in TokenMerge order (height and width even). */
int kdb_split_fac_grad(const float* y, const float* skip, const float* dup, float* out, int batch, int height, int width, int c, float* scratch,
                       void* stream);
/* class_emb's gradient: out[j, :] = sum over the rows r < rows with cls[r] == j (int64, device) of demb[r, :] (rows ldd >= mw floats apart),
 * rows in order, for every j < n_classes (zero where no row has that class; a class outside [0, n_classes) adds to nothing).  No scratch. */
int kdb_class_emb_grad(const float* demb, int64_t ldd, const int64_t* cls, float* out, int rows, int n_classes, int mw, void* stream);

/* C[M,N] = A[M,K] * W[N,K]^T, bf16 operands, fp32 accumulate (wgmma), bf16 out. */
int kdb_gemm_bf16(const void* a_bf16, const void* w_bf16, void* c_bf16, int M, int N, int K, void* stream);

/* out[M,N2/2] = value * gelu(gate) of A[M,K] * W_il[N2,K]^T: up_proj with the GEGLU fused in the epilogue
 * (image_transformer_v2.py:89-95,132-139).  W_il = up_proj.weight with its rows interleaved per 16-row group: 8 value rows
 * (rows g*8 .. g*8+7 of the first half) followed by the 8 matching gate rows (second half).  ss_in (may be NULL): [M, 8] fp32
 * sum(x^2) per 128-channel block of A's rows; the epilogue then scales the accumulator by 1/rms (fused RMSNorm). */
int kdb_gemm_bf16_geglu(const void* a_bf16, const void* w_il_bf16, void* c_bf16, int M, int N2, int K, const float* ss_in, void* stream);

/* The whole feed-forward block of a 128-wide level in one kernel, IN PLACE on the raw residual stream x[M,128] (bf16):
 *   x <- x + down_proj( value(x_n) * gelu(gate(x_n)) ),  x_n = x / rms(x)      (image_transformer_v2.py:479-493, :89-95; the AdaRMSNorm
 * channel scale is expected folded into w_up_il's columns).  w_up_il [2*d_ff,128] row-interleaved as for kdb_gemm_bf16_geglu,
 * w_down [128,d_ff]; ss_in [M,8] fp32 with sum(x^2) of each row in slot 0 (required), ss_out (may be NULL, may alias ss_in) receives
 * sum(x_new^2).  Needs M % 128 == 0, d_ff % 64 == 0, d_ff >= 192.  The [M,d_ff] hidden never leaves the SM. */
int kdb_ffn_fused_bf16(void* x_bf16, const void* w_up_il_bf16, const void* w_down_bf16, int M, int d_ff, const float* ss_in, float* ss_out,
                       void* stream);

/* The whole self-attention block of a 128-wide shifted-window level in one kernel, IN PLACE on the raw residual stream
 * x[batch,h,w,128] (bf16), two heads of d_head 64, window 8:
 *   x <- x + out_proj( window_attn( rope(cos_sim(q)), rope(cos_sim(k)), v ) ),  [q k v] = x_n . w_qkv^T,  x_n = x / rms(x)
 * (image_transformer_v2.py:253-337, :106-114, :187-199, :245-248, :396; the AdaRMSNorm channel scale is expected folded into w_qkv's
 * columns).  w_qkv [384,128] (feature order (t nh e)), w_out [128,128]; qk_scale [2] fp32 = the layer's `scale`; shift 0 or 4 (the
 * roll of the odd layers, :523).  rope: fp32 [2][8][h*w][4] = (cos t_2i, cos t_2i+1, sin t_2i, sin t_2i+1) of head n, pair i < 8 and
 * token y*w+x, where t_j (j < 16) is the RoPE angle of column j of a head (:245-248: pos_y * freqs[n][j] for j < 8, pos_x *
 * freqs[n][j-8] otherwise); column j < 16 of q and k rotates with column 16+j.  ss_in [batch*h*w,8] fp32 with sum(x^2) of each row
 * in slot 0 (required); ss_out (required, may alias ss_in) receives sum(x_new^2) in slot 0, slots 1..7 untouched.  Needs
 * h % 8 == 0 and w % 8 == 0.  q, k, v and the attention output never leave the SM. */
int kdb_attn_block_bf16(void* x_bf16, const void* w_qkv_bf16, const void* w_out_bf16, const float* rope, const float* qk_scale, int batch, int h,
                        int w, int shift, const float* ss_in, float* ss_out, void* stream);

/* out[B,h,w,nh*e] = attention(qkv[B,h,w,3*nh*e]) on fp32 or bf16 token tensors, feature order
 * (t nh e) as produced by qkv_proj (image_transformer_v2.py:377,386,422,431,467). q/k must already be
 * cosine-normalised and rotated.  attn_type/attn_param/shift as in KdbModelConfig (:523 for shift).
 * logit_bound (tensor-core path only, may be NULL): [n_heads] device floats, each in (0, 40], with |q . k| <= bound for that
 * head -- for cosine-similarity attention the layer's `scale` parameter (:106-114).  The kernels then use the bound as
 * softmax's fixed shift (one pass over the keys, no row maximum); NULL keeps the exact two-pass row-maximum kernels.
 * KDB_PREC_TF32 (fast 0, KDB_ATTN_GLOBAL, d_head 64, fp32 tensors, 1/sqrt(d_head) already in q): the image_v1 U-Net's attention
 * (layers.py:181-200) on the tensor cores, q, k, v and the probabilities truncated to tf32, fp32 accumulation, running-maximum softmax;
 * any other attention type, head size or `fast` at that precision is KDB_ERR_UNSUPPORTED.  KDB_PREC_FP16: the same with q, k, v and the
 * probabilities rounded to fp16 (nearest even); scores, softmax and the sum l of the rounded probabilities stay fp32. */
int kdb_attention(int precision, int fast, const void* qkv, void* out, int batch, int h, int w, int n_heads, int d_head,
                  int attn_type, int attn_param, int shift, const float* logit_bound, void* stream);

/* Derivatives of the fp32 kdb_attention (precision KDB_PREC_FP32, fast 0), the kernels the model's forward_jvp / forward_vjp launch.
 * qkv as for kdb_attention.
 *   kdb_attention_jvp: dout[B,h,w,nh*e] = the tangent of the attention output along dqkv (same layout as qkv).
 *   kdb_attention_vjp: out = kdb_attention's output on qkv, dout its gradient [B,h,w,nh*e] -> dqkv [B,h,w,3*nh*e], every element written.
 *                      stats: caller scratch of batch * n_heads * h * w * 3 floats (per-query softmax statistics).
 * A key set (query set for the VJP's per-key pass) too large for the kernels' shared memory returns KDB_ERR_UNSUPPORTED before any launch. */
int kdb_attention_jvp(const float* qkv, const float* dqkv, float* dout, int batch, int h, int w, int n_heads, int d_head,
                      int attn_type, int attn_param, int shift, void* stream);
int kdb_attention_vjp(const float* qkv, const float* out, const float* dout, float* dqkv, float* stats, int batch, int h, int w,
                      int n_heads, int d_head, int attn_type, int attn_param, int shift, void* stream);

/* The U-Net engine's fp32 convolution (ksize 1 or 3, zero padding ksize / 2, stride 1) as an implicit GEMM:
 *   out[m, n] = bias[n] + sum_{tap, c} w[n, tap, c] * in(pixel m shifted by tap, c) + resid[m, n]
 * Activations are token-major: in1 [batch, h, w, c1], in2 [batch, h, w, c2] (c2 = 0: one source; the input is the channel
 * concatenation of the two), out [batch, h, w, n_out].  w_tapmajor is [n_out, ksize*ksize, c1 + c2], the layout
 * kdb_unet_finalize derives from a torch weight [n_out, c1 + c2, ksize, ksize].  bias [n_out] may be NULL.  The residual
 * [batch, h, w, n_out] is the concatenation of r1 (rc1 channels) and r2 (n_out - rc1 channels): r1 NULL = none, rc1 = n_out
 * with r2 NULL = r1 alone.  c1, c2 and rc1 must be multiples of 4; batch * h * w is at most 65535 * 64 (KDB_ERR_BAD_SHAPE). */
int kdb_unet_conv(const float* in1, int c1, const float* in2, int c2, const float* w_tapmajor, const float* bias, const float* r1, int rc1,
                  const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream);

/* The backward kernels of kdb_unet_forward_train (fp32, deterministic, every output element written; arguments checked before any launch).
 * kdb_unet_conv_wgrad: the weight gradient of kdb_unet_conv in torch's layout, dw [n_out, c1 + c2, ksize, ksize] = sum over the pixels m of
 *   dy[m, n] (contiguous [batch, h, w, n_out]) times the input [in1 | in2] at pixel m shifted by the tap, zero outside the grid.  scratch:
 *   2^22 floats.
 * kdb_unet_flip_conv_weight: the weight of the input-gradient convolution, out [c_in, ksize^2, n_out] with out[c, tap, n] = w[n, ksize^2 - 1
 *   - tap, c] of a tap-major w [n_out, ksize^2, c_in]; kdb_unet_conv of dy with it is the input gradient (what kdb_unet_forward_train
 *   builds for every convolution).
 * kdb_unet_adagn_vjp: the backward of AdaGN (+ the erf GELU when gelu): x = [in1 | in2] [batch, hw, c1 + c2] the AdaGN input, dy its output
 *   gradient, the (weight, bias) pair read at cond + b * cond_batch_stride + ada_off as the forward reads it.  Writes dx (+ add when add is
 *   not NULL; add [batch, hw, c1 + c2] may alias neither output) to dx1 (c1 channels) and dx2 (c2), and the gradients of the weight and bias
 *   rows to dcond + b * dcond_batch_stride + ada_off (c1 + c2 floats each).
 * kdb_unet_resample_vjp: the adjoint of the 2x resampling of an h x w grid (h, w >= 2), reflect padding included: dout [batch, h/2, w/2, c]
 *   (up = 0) or [batch, 2h, 2w, c] (up = 1) -> din [batch, h, w, c] (+ add when not NULL; add may be din).
 * kdb_unet_mapping_vjp: the mapping network's backward of a finalized U-Net, one row per image: sigma [rows], aug_cond and mapping_cond as
 *   kdb_unet_conditioning takes them, dcond [rows, mapping_out] the gradient of the mapping network's output.  Writes, [rows, mapping_out]
 *   each, h0 (Fourier features + the mapping_cond Linear), a0 (the second Linear's input), dz0 and dz1 (the gradients of the two Linears'
 *   outputs) and dh0 (that of h0), and v [rows, mapping_cond_dim] (the mapping_cond vector, zeros where the model has none; v may be NULL
 *   when mapping_cond_dim is 0).  It needs (6 mapping_out + mapping_cond_dim) floats of shared memory, at most 48 KiB: a wider model
 *   returns KDB_ERR_UNSUPPORTED.
 * kdb_unet_proj_out_vjp: proj_out's input gradient, out [rows, k] = u [rows, n] w [n, k].
 * kdb_unet_unshuffle: pixel_unshuffle of an NCHW x [batch, c, h, w] (h, w multiples of p) to token rows out [batch (h/p) (w/p), ld], column
 *   (c, i, j) in torch's order; columns c p p .. ld - 1 are zero. */
int kdb_unet_conv_wgrad(const float* dy, int n_out, const float* in1, int c1, const float* in2, int c2, float* dw, int batch, int h, int w,
                        int ksize, float* scratch, void* stream);
int kdb_unet_adagn_vjp(const float* in1, int c1, const float* in2, int c2, const float* dy, const float* add, float* dx1, float* dx2,
                       const float* cond, int64_t cond_batch_stride, int ada_off, float* dcond, int64_t dcond_batch_stride, int groups, int gelu,
                       int batch, int hw, void* stream);
int kdb_unet_flip_conv_weight(const float* w_tapmajor, float* out, int n_out, int c_in, int ksize, void* stream);
int kdb_unet_resample_vjp(const float* dout, const float* add, float* din, int batch, int h, int w, int c, int up, void* stream);
int kdb_unet_mapping_vjp(const KdbUNet* m, int rows, const float* sigma, const float* aug_cond, const float* mapping_cond, const float* dcond,
                         float* h0, float* a0, float* dz0, float* dz1, float* dh0, float* v, void* stream);
int kdb_unet_proj_out_vjp(const float* u, const float* w, float* out, int64_t rows, int n, int k, void* stream);
int kdb_unet_unshuffle(const float* x, float* out, int batch, int c, int h, int w, int p, int ld, void* stream);

/* The reverse-mode kernels of kdb_model_forward_vjp / kdb_model_forward_train (fp32, deterministic: one writer per output element, no
 * atomics, two calls give the same bits; arguments checked before any launch).  Each takes the primal input of one op and the gradient of
 * its output, and writes (or, where named, adds to) the gradient of its input.
 * kdb_gemm_vjp: the input gradient of C = A W^T, dA [m, k] = dc [m, n] w [n, k] (n, k multiples of 4).  epi 0 (VJP_STORE) writes it to
 *   out [m, k]; epi 1 (VJP_UNPATCH_ACC) reads the rows as coarse tokens [m / (hc wc), hc, wc] and the columns as (nh nw e), e < cf (k = 4 cf),
 *   and ADDS each element to the fine token out [m / (hc wc), 2 hc, 2 wc, cf] it came from (the TokenMerge VJP).  m above 65535 * 64 runs as
 *   several launches of at most that many rows (of whole images for epi 1); one image of more rows is KDB_ERR_BAD_SHAPE.
 * kdb_rmsnorm_vjp: ADDS the input gradient of y = x rsqrt(mean(x^2) + 1e-6) s to dx: dx += r (s dy) - x r^3 mean(x s dy), x, dy, dx
 *   [rows, c]; the scale row of row i is scale + (i / rows_per_image) scale_bstride (scale_bstride 0: one shared row).
 * kdb_qknorm_rope_vjp: in place on the q and k thirds of dqkv [rows, 3, n_heads, d_head] (v is left alone): the backward of the cosine-sim
 *   scale and axial RoPE that kdb_model_forward applies to qkv (the primal before them, same layout), rows = batch t_tokens, pos [t_tokens, 2]
 *   (y, x), freqs [n_heads, r / 2], scale [n_heads], eps as the forward's (r = d_head / 2 and eps 1e-6 for image_transformer_v2; r = d_head
 *   for image_transformer_v1's layout).  dscale_rows (may be NULL): [rows, n_heads] the contribution of each (row, head) to the gradient of
 *   that head's scale.  d_head a multiple of 8, r of 4, r <= d_head.
 * kdb_geglu_vjp: h [m, 2f] = (value | gate) the up projection's output, dy [m, f] -> dh [m, 2f]: dy gelu(gate) | dy value gelu'(gate).
 * kdb_split_vjp_gather: TokenSplit's lerp backward on a fine grid of batch x height x width x c (height, width even): out [batch, height / 2,
 *   width / 2, 4 c] = fac dup gathered in TokenMerge order, and dup *= 1 - fac in place (fac: one device float).
 * kdb_split_unpatch_lerp: up [batch, height, width, c] = torch.lerp(skip, unpatch2x2(y), fac), y [batch, height / 2, width / 2, 4 c].
 * kdb_merge_scatter_add: dfine [batch, height, width, c] += unpatch2x2(d), d [batch, height / 2, width / 2, 4 c].
 * kdb_patch_out_vjp: the backward of out_norm + patch_out: dtokens [T, c0] (T = batch (height / patch_h) (width / patch_w)) =
 *   RMSNorm_vjp(tokens [T, c0], norm_scale [c0], patch(c_out u) w) with u [batch, channels, height, width] the output's gradient, w
 *   [patch_h patch_w channels, c0] and c_out Karras's (sigma [batch]) when sigma_data > 0, 1 otherwise.  dnorm (may be NULL): [T, c0] the
 *   gradient of out_norm's output; rstd (may be NULL): [T] each token's rsqrt(mean(x^2) + 1e-6).  It needs 4 (c0 + patch_h patch_w channels)
 *   floats of shared memory, at most 48 KiB: more returns KDB_ERR_UNSUPPORTED.
 * kdb_patch_in_vjp: grad_x [batch, channels, height, width] = unpatch(dtokens w) (dtokens [T, n], w [n, patch_h patch_w channels]); with
 *   sigma_data > 0, c_skip u + c_in unpatch(dtokens w), Karras's scalings of sigma [batch] and u the output's gradient.
 * kdb_model_mapping_vjp: the mapping network's backward of a finalized model, one row per image: sigma [rows], aug_cond, class_cond and
 *   mapping_cond as kdb_model_conditioning takes them, dcond [rows, mapping_width] the gradient of the mapping network's output.  With mw =
 *   mapping_width, D = mapping_depth, F = mapping_d_ff and F4 = F rounded up to a multiple of 4, each row of keep ((4 + D) mw + D (mw + 2 F +
 *   F4) floats) receives the forward's activations: the Fourier features of sigma at 0 and of aug_cond at mw, the summed embedding entering
 *   in_norm at 2 mw, the stream entering block l (l = D: out_norm) at (3 + l) mw, then per block l at (4 + D) mw + l (mw + 2 F + F4) its normed
 *   input (mw), up_proj output (2 F) and GEGLU output (F).  Each row of grad ((D + 2) mw + D (mw + 2 F) floats) receives the gradients: of
 *   the stream entering block l at l mw (l <= D), of block l's normed input at (D + 1) mw + l (mw + 2 F) and of its up_proj output
 *   mw later, and of the summed embedding at (D + 1) mw + D (mw + 2 F).  D <= 8, mw a multiple of 4; a network whose (mapping_cond_dim
 *   rounded up to 4) + 32 + F floats exceed 48 KiB of shared memory returns KDB_ERR_UNSUPPORTED. */
int kdb_gemm_vjp(const float* dc, const float* w, float* out, int64_t m, int n, int k, int epi, int hc, int wc, int cf, void* stream);
int kdb_rmsnorm_vjp(const float* x, const float* dy, float* dx, const float* scale, int64_t scale_bstride, int64_t rows_per_image, int64_t rows,
                    int c, void* stream);
int kdb_qknorm_rope_vjp(const float* qkv, float* dqkv, const float* pos, const float* freqs, const float* scale, float eps, int r, int64_t rows,
                        int t_tokens, int n_heads, int d_head, float* dscale_rows, void* stream);
int kdb_geglu_vjp(const float* h, const float* dy, float* dh, int64_t m, int f, void* stream);
int kdb_split_vjp_gather(float* dup, float* out, const float* fac, int batch, int height, int width, int c, void* stream);
int kdb_split_unpatch_lerp(const float* y, const float* skip, const float* fac, float* up, int batch, int height, int width, int c, void* stream);
int kdb_merge_scatter_add(const float* d, float* dfine, int batch, int height, int width, int c, void* stream);
int kdb_patch_out_vjp(const float* tokens, const float* norm_scale, const float* w, const float* u, const float* sigma, float sigma_data,
                      float* dtokens, int batch, int channels, int height, int width, int patch_h, int patch_w, int c0, float* dnorm, float* rstd,
                      void* stream);
int kdb_patch_in_vjp(const float* dtokens, const float* w, const float* u, const float* sigma, float sigma_data, float* grad_x, int batch,
                     int channels, int height, int width, int patch_h, int patch_w, int n, void* stream);
int kdb_model_mapping_vjp(const KdbModel* m, int rows, const float* sigma, const float* aug_cond, const int64_t* class_cond,
                          const float* mapping_cond, const float* dcond, float* keep, float* grad, void* stream);

/* The same convolution, arguments and layouts on the tensor cores (wgmma, the kernel kdb_unet_forward runs at KDB_PREC_TF32): the
 * products take tf32 operands -- the low 13 mantissa bits of every input and weight element are ignored (truncation), so a caller
 * wanting round-to-nearest weights rounds them first, as kdb_unet_finalize does -- and accumulate in fp32; bias and residual are added
 * in fp32.  No grid-row limit on batch * h * w. */
int kdb_unet_conv_tf32(const float* in1, int c1, const float* in2, int c2, const float* w_tapmajor, const float* bias, const float* r1,
                       int rc1, const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream);

/* The same convolution and arguments with fp16 operands (wgmma, the kernel kdb_unet_forward runs at KDB_PREC_FP16).  w_tapmajor_f16 is
 * the tap-major weight in fp16, [n_out, ksize*ksize, ld] with ld = c1 + c2 rounded up to a multiple of 8 (the padding channels are
 * never read), as kdb_unet_finalize rounds it (nearest even).  The activations are rounded to the nearest fp16 (ties to even) inside
 * the kernel, without saturation: an input of magnitude >= 65520 becomes +-inf there and reaches the outputs it feeds as inf or NaN.
 * Products accumulate in fp32; bias and residual are added in fp32.  No grid-row limit on batch * h * w. */
int kdb_unet_conv_fp16(const float* in1, int c1, const float* in2, int c2, const void* w_tapmajor_f16, const float* bias, const float* r1,
                       int rc1, const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream);

/* ------------------------------------------------------------------------------------------
 * Sample scoring: KID and FID on extracted features (evaluation.py:93-161), fp32 FFMA products as the reference computes them with
 * TF32 off.  Features are row-major fp32 [rows, d].  No atomics: two calls on the same inputs return the same bits.  Unlike the
 * solver and forward calls these are not meant for CUDA-graph capture (kdb_mmd_sums copies its segment list from host memory).
 * ------------------------------------------------------------------------------------------ */

/* Squared MMD with the polynomial kernel k(a, b) = (a . b / d + 1)^3 of S segments in one call: segment s pairs rows
 * [x_offsets_host[s], x_offsets_host[s + 1]) of x [m, d] with rows [y_offsets_host[s], y_offsets_host[s + 1]) of y [n, d] (kid's
 * partitions, evaluation.py:114-123, or the leading batch entries of squared_mmd, :99-111).  out [S, 4] fp64 receives per segment the
 * sum of k(x, x) off its diagonal, the same of k(y, y), the sum of k(x, y) and term_1 + term_2 - term_3 formed in fp64 (nan for a
 * segment of fewer than 2 rows, as 0/0 in the reference).  Each kernel value is an fp32 dot product over d (fmaf in index order), then
 * fp32 (dot / d + 1)^3; only the tiles on or above the diagonal of k(x, x) and k(y, y) are computed and the strict upper triangle counts
 * twice; tile sums and their totals are fp64 in a fixed order.  Offsets are host arrays of S + 1 nondecreasing row indices within
 * [0, m] / [0, n], 1 <= S <= 65535.  kdb_mmd_workspace_bytes returns the workspace the same segment list needs (or a negative
 * KDB_ERR_*); a shorter one returns KDB_ERR_WORKSPACE.  Two launches whatever S is. */
int64_t kdb_mmd_workspace_bytes(const int64_t* x_offsets_host, const int64_t* y_offsets_host, int n_segments);
int kdb_mmd_sums(const float* x, int64_t m, const float* y, int64_t n, int d, const int64_t* x_offsets_host, const int64_t* y_offsets_host,
                 int n_segments, double* out, void* workspace, size_t workspace_bytes, void* stream);

/* out [batch, m, n] fp32 = (x . y^T / d + 1)^3 of x [batch, m, d] and y [batch, n, d] (evaluation.py:93-96), each element as
 * kdb_mmd_sums computes it.  batch <= 65535 and ceil(m / 64) <= 65535. */
int kdb_polynomial_kernel(const float* x, const float* y, float* out, int batch, int m, int n, int d, void* stream);

/* mean [d] and cov [d, d] fp32 of x [n, d] (evaluation.py:151-155: x.mean(0) and torch.cov(x.T)): the column sums in fp64 in a fixed
 * order, divided by n; then the upper-triangle 64x64 tiles of (x - mean)^T (x - mean) / (n - 1), with x - mean in fp32 and fmaf over the
 * samples in order, each element written to (i, j) and (j, i), so cov is exactly symmetric (n = 1 gives nan, as torch.cov).
 * 1 <= n <= INT32_MAX.  Two launches, no workspace. */
int kdb_feature_mean_cov(const float* x, int64_t n, int d, float* mean, float* cov, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training loop: the EMA model update after each optimizer step (utils.py:88-104 ema_update)
 * ------------------------------------------------------------------------------------------ */

/* One segment of kdb_ema_update: n fp32 elements at src and dst (device, 4-byte aligned, not overlapping).
 * KDB_EMA_LERP (a parameter): dst = torch.lerp(dst, src, weight); KDB_EMA_COPY (a buffer): dst = src. */
#define KDB_EMA_LERP 0
#define KDB_EMA_COPY 1
typedef struct KdbEmaSeg {
  const float* src;
  float* dst;
  int64_t n;
  int32_t mode;
} KdbEmaSeg;

/* Every segment of the host table segs_host[0 .. n_segs) in one launch, weight = 1 - decay.  The lerp is torch's CUDA lerp_ with a scalar
 * weight, |w| < 0.5 ? dst + w (src - dst) : src - (src - dst) (1 - w) in fp32, each branch one fused multiply-add: bit for bit lerp_ on the
 * same GPU.  A segment of n = 0 is skipped; NULL src or dst with n > 0, a mode other than KDB_EMA_LERP / KDB_EMA_COPY or a pointer that
 * is not 4-byte aligned return KDB_ERR_BAD_ARG before any CUDA call.  Grid-stride over all segments' elements, 128-bit loads and stores
 * where src and dst are co-aligned (scalar head and tail), scalar otherwise; every element written once, no atomics.  The table is staged
 * in a pinned host buffer the library reuses and copied to the device on `stream`, so the call is not capturable: under CUDA-graph capture
 * it returns KDB_ERR_UNSUPPORTED.  The library's first call on a device, and a call with more segments than any before, allocates. */
int kdb_ema_update(const KdbEmaSeg* segs_host, int n_segs, float weight, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training data: KarrasAugmentationPipeline (augmentation.py:32-89) for a batch, one launch
 * ------------------------------------------------------------------------------------------ */

/* images [B, C, H, W] uint8; draws [B, 13] fp32, each image's scalar draws in the reference's order (randint(2), rand, randint(2),
 * rand, randn, rand, rand, rand, rand, randn, rand, randn, randn; randint as 0 or 1).  Writes image_orig = x / 255 * 2 - 1 (bit for bit
 * the reference's), cond [B, 9] and image [B, C, H, W]: the affine warp of x / 255 by the reference's matrix, bicubic (Catmull-Rom)
 * with numpy's 'reflect' border, unclipped, * 2 - 1.  The matrix is formed in fp32 from the draws as the reference's torch ops form it
 * (a gate is `draw < a_prob` in fp32; h, w of the reference are W, H) and inverted in fp64; `mat` (may be NULL) receives it, [B, 9].
 * disable_all != 0 copies image_orig to image and zeroes cond.  NULL images, draws, image, image_orig or cond return KDB_ERR_BAD_ARG,
 * B, C, H or W < 1 KDB_ERR_BAD_SHAPE, a non-finite a_scale, a_aniso or a_trans KDB_ERR_BAD_ARG, all before any CUDA call.  Every
 * output written once, deterministic, no workspace. */
int kdb_augment(const uint8_t* images, const float* draws, int B, int C, int H, int W, float a_prob, double a_scale, double a_aniso,
                double a_trans, int disable_all, float* image, float* image_orig, float* cond, float* mat, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KDIFFUSION_B200_H */
