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

#define KDB_ABI_VERSION 7

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

/* Counter-based standard-normal fill (Philox4x32-10 + Box-Muller): element i of sample b gets the
 * (seed[b], stream_id, i) variate, so results do not depend on how a batch is sharded across GPUs.
 * Replaces torch.randn_like in default_noise_sampler (sampling.py:61-62).  seeds is a device int64 [B]. */
int kdb_noise_normal(float* out, const int64_t* seeds, uint64_t stream_id, int batch, int64_t per_sample,
                     void* stream);

/* Virtual Brownian bridge increment W(t1) - W(t0), normalised by sqrt(|t1 - t0|), per sample.
 * Replaces BatchedBrownianTree / BrownianTreeNoiseSampler (sampling.py:65-114): dyadic Brownian-bridge
 * tree on [t_min, t_max] of `depth` levels evaluated from (seed[b], node, element) counters.
 * Parity with torchsde is UNPINNED (torchsde absent); contract = determinism, additivity, unit variance. */
int kdb_noise_brownian(float* out, const int64_t* seeds, int batch, int64_t per_sample,
                       double t_min, double t_max, double t0, double t1, int depth, void* stream);

/* ------------------------------------------------------------------------------------------
 * image_transformer_v2 denoiser engine (models/image_transformer_v2.py:667-762, layers.py:45-90)
 * ------------------------------------------------------------------------------------------ */

#define KDB_MAX_LEVELS 8

enum { KDB_ATTN_NONE = 0, KDB_ATTN_GLOBAL = 1, KDB_ATTN_NEIGHBORHOOD = 2, KDB_ATTN_SHIFTED_WINDOW = 3 };
enum { KDB_PREC_FP32 = 0, KDB_PREC_BF16 = 1 };   /* arithmetic of the token stream / GEMM operands */

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
} KdbModelConfig;

typedef struct KdbModel KdbModel;

int  kdb_model_create(const KdbModelConfig* cfg, KdbModel** out);
void kdb_model_destroy(KdbModel* m);

/* Bind one state-dict entry (fp32, contiguous, device) by its reference key name, e.g.
 * "down_levels.0.1.self_attn.qkv_proj.weight" (key list: SURVEY.md section 8b).  The pointer is
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

/* Debug/parity tap: arm a copy of one intermediate of the NEXT forward into `out` (fp32, device).
 * name: "patch_in", "L<l>.down", "L<l>.merge", "mid", "L<l>.split", "L<l>.up", "layer<k>.xn1",
 * "layer<k>.qkv", "layer<k>.ao", "layer<k>.attn", "layer<k>.ff" (k = execution order).
 * After the forward, kdb_model_tap_count returns the number of floats written (0 = name never hit,
 * <0 = capacity too small).  The tap disarms itself after one forward. */
int     kdb_model_debug_tap(KdbModel* m, const char* name, float* out, int64_t capacity);
int64_t kdb_model_tap_count(const KdbModel* m);

/* ------------------------------------------------------------------------------------------
 * Stand-alone kernels exposed for unit tests / profiling (same code the engine launches)
 * ------------------------------------------------------------------------------------------ */

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

/* out[B,h,w,nh*e] = attention(qkv[B,h,w,3*nh*e]) on fp32 or bf16 token tensors, feature order
 * (t nh e) as produced by qkv_proj (image_transformer_v2.py:377,386,422,431,467). q/k must already be
 * cosine-normalised and rotated.  attn_type/attn_param/shift as in KdbModelConfig (:523 for shift).
 * logit_bound (tensor-core path only, may be NULL): [n_heads] device floats, each in (0, 40], with |q . k| <= bound for that
 * head -- for cosine-similarity attention the layer's `scale` parameter (:106-114).  The kernels then use the bound as
 * softmax's fixed shift (one pass over the keys, no row maximum); NULL keeps the exact two-pass row-maximum kernels. */
int kdb_attention(int precision, int fast, const void* qkv, void* out, int batch, int h, int w, int n_heads, int d_head,
                  int attn_type, int attn_param, int shift, const float* logit_bound, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KDIFFUSION_B200_H */
