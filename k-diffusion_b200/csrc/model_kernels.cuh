// model_kernels.cuh -- launchers for the per-op kernels of the image_transformer_v2 forward pass.
// "generic" kernels are precision-templated SIMT kernels (fp32 = the exact path used for the
// rtol 1e-3 / atol 1e-5 parity gate; bf16 = fallback for shapes the tensor-core kernels do not cover).
#pragma once
#include "common.cuh"

namespace kdb {

// The epilogue of a token-stream GEMM.  The values are gemm_wg_kernel's EPI template argument; the SIMT GEMM runs STORE, RESID and
// SPLIT_LERP only.
enum GemmEpilogue { EPI_STORE = 0, EPI_RESID = 1, EPI_GEGLU = 2, EPI_SPLIT_LERP = 3, EPI_QKV_ROPE = 4, EPI_PATCH_OUT = 5 };

struct GemmEpi {
  int mode = EPI_STORE;
  // EPI_GEGLU (tensor-core path only): the rows of W interleave 8 value / 8 gate rows; out[M, N/2] = value * gelu(gate)
  const void* resid = nullptr;   // EPI_RESID: [M,N] same type as out.  EPI_SPLIT_LERP: skip [B, 2hc, 2wc, C]
  const float* fac = nullptr;    // EPI_SPLIT_LERP: device scalar (TokenSplit.fac)
  int hc = 0, wc = 0, C = 0;     // EPI_SPLIT_LERP: coarse grid and fine channel count (N == 4*C)
  // EPI_QKV_ROPE (tensor-core path only): cosine-sim scaling + axial RoPE of the q and k thirds (N == 3*C, d_head 64)
  const float2* rope = nullptr;  // launch_rope_table: float4 [nh][rope_r / 4][T_tokens] = (cos, cos, sin, sin) of the angle pairs
  const float* qk_scale = nullptr;   // [nh]
  float qk_eps = 1e-6f;          // QkRope::eps (image_transformer_v2's unless set)
  int rope_r = 32;               // QkRope::R: 32 (image_transformer_v2) or 64 (image_transformer_v1, all of a head)
  int nh = 0, T_tokens = 0;
  // TokenMerge folded into the A-operand load (tensor-core path only): A = fine tokens [B, 2*mhc, 2*mwc, mC], K = 4*mC in
  // (nh nw e) order, M = B*mhc*mwc.  mC == 0 -> A is a plain [M, K] matrix.
  int mhc = 0, mwc = 0, mC = 0;
  // fused RMSNorm (tensor-core kernel only).  Consumer (EPI_STORE / EPI_QKV_ROPE / EPI_GEGLU / EPI_PATCH_OUT): A is the raw
  // residual stream, W already carries the channel scale, ss_in [M, 8] holds sum(x^2) per 128-channel block of every row and the
  // epilogue scales the accumulator by 1/rms (q/k thirds of EPI_QKV_ROPE are scale invariant).  Producer (EPI_RESID /
  // EPI_SPLIT_LERP, and EPI_STORE): ss_out receives those sums for the rows written.
  const float* ss_in = nullptr;
  float* ss_out = nullptr;
  // EPI_PATCH_OUT (tensor-core path only): rows are the tokens [B, H/4, W/4], columns the 4x4 patches of 3 channels (48 of N = 64
  // used).  The GEMM's bf16 output is unused: the epilogue un-patches to img, fp32 NCHW [B, 3, H, W], and with sigma_data > 0
  // applies the Karras combine with x_in [B, 3, H, W] and sigma [B].
  float* img = nullptr;
  const float* x_in = nullptr;
  const float* sigma = nullptr;
  float sigma_data = 0.f;
  int H = 0, W = 0;
};

// NCHW offset of patch column n = (nh, nw, c) of token (ty, tx) of image b: channel c of pixel (ty ph + nh, tx pw + nw)
__device__ __forceinline__ int64_t patch_pixel(int b, int ty, int tx, int n, int C, int H, int W, int ph, int pw) {
  const int q = n / C, c = n - q * C;
  const int nh = q / pw, nw = q - nh * pw;
  return nchw_offset(b, c, ty * ph + nh, tx * pw + nw, C, H, W);
}

// TokenMerge / TokenSplit 2x2 order (image_transformer_v2.py:594,618): channel e of quadrant q = 2 nh + nw of coarse token (hy, wx)
// of image b is channel e of fine token (2 hy + nh, 2 wx + nw) of [B, 2 hc, 2 wc, Cf]
__device__ __forceinline__ int64_t fine_offset(int64_t b, int hy, int wx, int q, int e, int hc, int wc, int Cf) {
  return ((b * (2 * hc) + (2 * hy + (q >> 1))) * (2 * wc) + (2 * wx + (q & 1))) * Cf + e;
}
// element i of a coarse [B, hc, wc, 4 Cf] tensor in that order -> offset of its fine element
__device__ __forceinline__ int64_t merge_source(int64_t i, int hc, int wc, int Cf) {
  const int e = (int)(i % Cf);
  int64_t r = i / Cf;
  const int q = (int)(r & 3);
  r >>= 2;
  const int wx = (int)(r % wc);
  r /= wc;
  const int hy = (int)(r % hc);
  return fine_offset(r / hc, hy, wx, q, e, hc, wc, Cf);
}

// x [B,C,H,W] fp32 (* c_in(sigma) if sigma_data > 0) -> tokens [B, H/ph, W/pw, N]   (image_transformer_v2.py:586-595,723-724)
template <typename T>
int launch_patch_in(const float* x, const float* sigma, float sigma_data, const float* W, T* out, int B, int C, int H, int Wd,
                    int ph, int pw, int N, cudaStream_t st);

// y = x * rsqrt(mean(x^2) + eps) * scale      (image_transformer_v2.py:98-103,152,166)
// scale row for token row r: scale + (r / rows_per_batch) * scale_bstride
template <typename T>
int launch_rmsnorm(const T* x, T* y, const float* scale, int64_t scale_bstride, int64_t rows_per_batch, int64_t rows, int C,
                   cudaStream_t st);

// C[M,N] = A[M,K] W[N,K]^T with epilogue (nn.Linear bias=False, image_transformer_v2.py:126-129)
template <typename T, typename TW>
int launch_gemm_simt(const T* A, const TW* W, T* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st);

// Cosine-sim scaling and axial RoPE of one layer's q and k heads of e columns (image_transformer_v2.py:106-114,187-199,245-248):
//   q^ = sqrt(scale_h) q / sqrt(sum q^2 + eps), then column j < R/2 of q^ and column j + R/2 turn by theta_j = pos_y freqs[h, j]
//   (j < R/4) or pos_x freqs[h, j] (j >= R/4); columns from R on pass through.
// image_transformer_v2: R = e/2, freqs = (f, f) of its pos_emb.freqs f [nh, e/8], eps 1e-6.  image_transformer_v1 (QKNorm + the
// interleaved AxialRoPE of all e columns) is the same map on q, k rows permuted by kdb_model_finalize: R = e, freqs = exp(freqs_h) |
// exp(freqs_w), scale = exp(min(qk_norm.scale, ln 100)), eps = e * 1e-6.
struct QkRope {
  const float* freqs = nullptr;   // [nh, R/2]
  const float* scale = nullptr;   // [nh]; |q^ . k^| <= scale_h
  float eps = 0.f;
  int R = 0;
};

// QkRope on qkv [rows, 3, nh, e] src -> dst (src == dst: in place; else v is copied through).  pos [T,2] (y,x) for the level; rows = B*T
template <typename T>
int launch_qknorm_rope(const T* src, T* dst, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e, cudaStream_t st);

// softmax(q k^T) v over the key set of attn_type (scale 1.0); qkv [B,h,w,3,nh,e] -> out [B,h,w,nh,e]
template <typename T>
int launch_attention_generic(const T* qkv, T* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                             cudaStream_t st);

// out[M,F] = h[M,0:F] * gelu_erf(h[M,F:2F])     (image_transformer_v2.py:89-95)
template <typename T>
int launch_geglu(const T* h, T* out, int64_t M, int F, cudaStream_t st);

// TokenMerge 2x2 gather: x [B,H,W,C] -> [B,H/2,W/2,(nh nw e)]   (image_transformer_v2.py:594)
template <typename T>
int launch_merge_gather(const T* x, T* out, int B, int H, int Wd, int C, cudaStream_t st);

// out_norm (RMSNorm) + patch_out Linear + un-patch to NCHW + optional Karras combine with x_in
// (image_transformer_v2.py:598-607,758-760; layers.py:88-90)
template <typename T>
int launch_patch_out(const T* tokens, const float* norm_scale, const float* W, const float* x_in, const float* sigma,
                     float sigma_data, float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st);

// Tangent kernels of the forward-mode derivative (fp32).  Each takes the primal input of one nonlinear op and its tangent and
// writes the tangent of the output; the primal op is launched separately, unchanged.
// RMSNorm: dy = s (r dx - x r^3 mean(x dx)), r = rsqrt(mean(x^2) + eps); scale rows as launch_rmsnorm
int launch_rmsnorm_jvp(const float* x, const float* dx, float* dy, const float* scale, int64_t scale_bstride, int64_t rows_per_batch,
                       int64_t rows, int C, cudaStream_t st);
// cosine-sim scale + RoPE of the tangent q, k (in place on dqkv [rows, 3, nh, e]); qkv holds the primal q, k BEFORE launch_qknorm_rope
int launch_qknorm_rope_jvp(const float* qkv, float* dqkv, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e,
                           cudaStream_t st);
// attention tangent over the key set of launch_attention_generic; qkv = the normalised, rotated primal, dqkv its tangent
int launch_attention_jvp(const float* qkv, const float* dqkv, float* dout, int B, int h, int w, int nh, int e, int attn_type, int attn_param,
                         int shift, cudaStream_t st);
// GEGLU tangent: dout = da gelu(g) + a gelu'(g) dg over h / dh [M, 2F]
int launch_geglu_jvp(const float* h, const float* dh, float* dout, int64_t M, int F, cudaStream_t st);
// out_norm tangent + patch_out + un-patch; sigma_data > 0: out = c_skip v + c_out dF, else dF
int launch_patch_out_jvp(const float* tokens, const float* dtokens, const float* norm_scale, const float* W, const float* v_in, const float* sigma,
                         float sigma_data, float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st);

// Backward kernels of the reverse-mode derivative (fp32).  Each takes the primal input of one op (recomputed from the tape by the op's
// forward launch) and the gradient of its output, and writes (or, where named, adds) the gradient of its input.  No atomics.
enum GemmVjpEpilogue { VJP_STORE = 0, VJP_UNPATCH_ACC = 1 };
// dA[M,K] = dC[M,N] W[N,K], the input gradient of C = A W^T, W read along N (no transposed copy).  VJP_UNPATCH_ACC: rows are coarse
// tokens of [B, hc, wc], columns (nh nw e) with e < Cf; the result is ADDED to the fine tokens out [B, 2hc, 2wc, Cf] (TokenMerge VJP)
int launch_gemm_vjp(const float* dC, const float* W, float* out, int64_t M, int N, int K, int epi, int hc, int wc, int Cf, cudaStream_t st);
// RMSNorm: dx += r (s dy) - x r^3 mean(x s dy), r = rsqrt(mean(x^2) + eps); scale rows as launch_rmsnorm
int launch_rmsnorm_vjp(const float* x, const float* dy, float* dx, const float* scale, int64_t scale_bstride, int64_t rows_per_batch,
                       int64_t rows, int C, cudaStream_t st);
// cosine-sim scale + RoPE, in place on the q, k thirds of dqkv [rows, 3, nh, e] (v passes through); qkv = the primal BEFORE launch_qknorm_rope.
// dscale_rows != nullptr: also [rows, nh] the contribution of each (row, head) to the gradient of the head's scale
int launch_qknorm_rope_vjp(const float* qkv, float* dqkv, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e,
                           cudaStream_t st, float* dscale_rows = nullptr);
// attention over the key set of launch_attention_generic: qkv the normalised, rotated primal, out its output, dout the output gradient
// -> dqkv [B, T, 3, nh, e].  stats: scratch of B * nh * T * 3 floats (per-query softmax statistics handed from the query-centric pass
// to the key-centric one)
int launch_attention_vjp(const float* qkv, const float* out, const float* dout, float* dqkv, float* stats, int B, int h, int w, int nh, int e,
                         int attn_type, int attn_param, int shift, cudaStream_t st);
// GEGLU: h [M, 2F] primal up_proj output, dy [M, F] -> dh [M, 2F]
int launch_geglu_vjp(const float* h, const float* dy, float* dh, int64_t M, int F, cudaStream_t st);
// TokenSplit lerp: out [B, H/2, W/2, 4C] = patch2x2(fac dup) (then launch_gemm_vjp with the split weight), dup *= (1 - fac) in place
int launch_split_vjp_gather(float* dup, float* out, const float* fac, int B, int H, int Wd, int C, cudaStream_t st);
// The elementwise halves of TokenSplit and of the TokenMerge VJP around a plain [M, N] GEMM (the tf32 training route): H, Wd the fine grid, C
// the fine channels.  up = lerp(skip, unpatch2x2(y), fac) with y [B, H/2, W/2, 4C]; dfine += unpatch2x2(d) with d [B, H/2, W/2, 4C].
int launch_split_unpatch_lerp(const float* y, const float* skip, const float* fac, float* up, int B, int H, int Wd, int C, cudaStream_t st);
int launch_merge_scatter_add(const float* d, float* dfine, int B, int H, int Wd, int C, cudaStream_t st);
// out_norm + patch_out + un-patch: dtokens = RMSNorm_vjp(tokens, patch(c_out u) W_po)  (c_out = 1 when sigma_data <= 0)
// Where given, also dnorm [tokens, C0] the gradient of out_norm's output and rstd [tokens] each token's rsqrt(mean(x^2) + eps) as the
// forward computes it
int launch_patch_out_vjp(const float* tokens, const float* norm_scale, const float* W, const float* u, const float* sigma, float sigma_data,
                         float* dtokens, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st, float* dnorm = nullptr,
                         float* rstd = nullptr);
// patch_in: grad_x = c_skip u + c_in unpatch(dtokens W_pi) (sigma_data > 0), else unpatch(dtokens W_pi)
int launch_patch_in_vjp(const float* dtokens, const float* W, const float* u, const float* sigma, float sigma_data, float* grad_x, int B, int C,
                        int H, int Wd, int ph, int pw, int N, cudaStream_t st);

// tiled fast variants (patch_kernels.cu); return false when the shape is outside their envelope
template <typename T>
bool launch_patch_in_tiled(const float* x, const float* sigma, float sigma_data, const float* W, T* out, int B, int C, int H, int Wd, int ph,
                           int pw, int N, cudaStream_t st, int* rc);
template <typename T>
bool launch_patch_out_tiled(const T* tokens, const float* norm_scale, const float* W, const float* x_in, const float* sigma, float sigma_data,
                            float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st, int* rc);

// mapping network + concatenated AdaRMSNorm projections (image_transformer_v2.py:552-581,734-740,166)
struct CondWeights {
  int mw, depth, dff, n_classes, mcond_dim, ada_total;
  const float *time_emb, *time_in, *aug_emb, *aug_in, *class_emb, *mcond_in;
  const float *in_norm, *out_norm;
  const float* blk_norm[8];
  const float* blk_up[8];
  const float* blk_down[8];
  const float* ada_cat;     // [ada_total, mw]
};
int launch_conditioning(const CondWeights& w, int rows, const float* sigma, const float* aug, const int64_t* cls, const float* mcond,
                        float* out, int64_t out_stride, cudaStream_t st);

// The mapping network's backward, one CTA per conditioning row (train_kernels.cu reduces what it leaves into the weight gradients).
// Per row it recomputes the forward of launch_conditioning into `keep` and, from dcond [rows, mw] (the gradient of the mapping network's
// output), writes the gradients of the activations into `grad`.  MapLayout gives the offsets of each vector in a row of either.
struct MapLayout {
  int mw, dff, depth;
  // keep: Fourier features of sigma and of aug_cond, the summed embedding entering in_norm, the stream r[l] entering block l (r[depth]:
  // entering out_norm), each block's normed input, up_proj output (value | gate) and GEGLU output
  __host__ __device__ int ff_t() const { return 0; }
  __host__ __device__ int ff_a() const { return mw; }
  __host__ __device__ int emb() const { return 2 * mw; }
  __host__ __device__ int r(int l) const { return 3 * mw + l * mw; }
  __host__ __device__ int xn(int l) const { return r(depth + 1) + l * blk(); }
  __host__ __device__ int up(int l) const { return xn(l) + mw; }
  __host__ __device__ int g(int l) const { return up(l) + 2 * dff; }
  __host__ __device__ int blk() const { return mw + 2 * dff + ((dff + 3) & ~3); }
  __host__ __device__ int keep_floats() const { return xn(depth); }
  // grad: d r[l] (l <= depth), d(normed input) and d(up_proj output) of block l, d(embedding entering in_norm)
  __host__ __device__ int dr(int l) const { return l * mw; }
  __host__ __device__ int dxn(int l) const { return (depth + 1) * mw + l * (mw + 2 * dff); }
  __host__ __device__ int dh(int l) const { return dxn(l) + mw; }
  __host__ __device__ int demb() const { return dxn(depth); }
  __host__ __device__ int grad_floats() const { return demb() + mw; }
};
int launch_mapping_backward(const CondWeights& w, int rows, const float* sigma, const float* aug, const int64_t* cls, const float* mcond,
                            const float* dcond, float* keep, float* grad, cudaStream_t st);

// Parameter-gradient reductions (train_kernels.cu), fp32.  No atomics; every sum runs in an order fixed by the shapes alone, so two calls
// give the same bits.  `part` is scratch of kTrainPartFloats floats (reduction partials).  A NULL output skips the launch.
constexpr int64_t kTrainPartFloats = int64_t(1) << 22;
// dW[N, K] = sum over the rows m < M of dY[m, n] X[m, k] (the weight gradient of Y = X W^T); dY and X rows ldy, ldx floats apart
int launch_wgrad(const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, int64_t M, int N, int K, float* part, cudaStream_t st);
// the same with X the TokenMerge gather of the fine tokens [B, 2hc, 2wc, Cf] (M = B hc wc coarse rows, K = 4 Cf) read in place
int launch_wgrad_merge(const float* dY, int64_t ldy, const float* fine, float* dW, int64_t M, int N, int hc, int wc, int Cf, float* part,
                       cudaStream_t st);
// Both with tf32 operands on the tensor cores (mma.sync): dY and X truncated to tf32 (the low 13 mantissa bits cleared), fp32 accumulation,
// the same row chunks and chunk-order sum as launch_wgrad
int launch_wgrad_tf32(const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, int64_t M, int N, int K, float* part,
                      cudaStream_t st);
int launch_wgrad_tf32_merge(const float* dY, int64_t ldy, const float* fine, float* dW, int64_t M, int N, int hc, int wc, int Cf, float* part,
                            cudaStream_t st);
// out[b * ldo + c] = sum over the rows r of image b of dy[r, c] x[r, c] rsqrt(mean(x_r^2) + eps): the gradient of an RMSNorm's channel scale
// per image (rows_per_batch rows each; rows_per_batch == rows: one sum over all rows)
int launch_norm_scale_grad(const float* x, int64_t ldx, const float* dy, int64_t ldy, float* out, int64_t ldo, int64_t rows_per_batch,
                           int64_t rows, int C, float* part, cudaStream_t st);
// out[c] = sum over r < rows of P[r, c]
int launch_colsum(const float* P, int64_t rows, int C, float* out, float* part, cudaStream_t st);
// the gradient of TokenSplit's fac: sum of (y - skip) dup, y [B, H/2, W/2, 4C] the split projection in TokenMerge order, skip and dup
// (the gradient of the split's output) [B, H, W, C]
int launch_split_fac_grad(const float* y, const float* skip, const float* dup, float* out, int B, int H, int Wd, int C, float* part,
                          cudaStream_t st);
// patch_in's weight gradient: dW [N, (nh nw c)] = sum over tokens of dtok[tok, n] times the patch row of the NCHW image x [B, C, H, W],
// read in place
int launch_wgrad_patch_in(const float* dtok, const float* x, float* dW, int B, int C, int H, int Wd, int ph, int pw, int N, float* part,
                          cudaStream_t st);
// patch_out's weight gradient: dW [(nh nw c), C0] = sum over tokens of the patch row of u [B, C, H, W] times out_norm's output, both read
// in place (the output as tokens [B T, C0] * (scale * rstd), rstd from launch_patch_out_vjp)
int launch_wgrad_patch_out(const float* u, const float* tokens, const float* scale, const float* rstd, float* dW, int B, int C, int H, int Wd,
                           int ph, int pw, int C0, float* part, cudaStream_t st);
// class_emb's gradient: out[k, :] = sum over the rows r with cls[r] == k of demb[r, :] (ld ldd), rows in order; every row k < n_classes written
int launch_class_emb_grad(const float* demb, int64_t ldd, const int64_t* cls, float* out, int rows, int n_classes, int mw, cudaStream_t st);
// DenoiserWithVariance's loss (layers.py:93-101), one CTA per image of n elements: with r = f - (x - c_skip xn) / c_out, xn = x + noise sigma,
// and m = mean(r^2) (a fixed-order block sum in double), loss[b] = (m e^-lv + lv) / 2 and dlogvar[b] = (1 - m e^-lv) / 2 (or NULL) formed in
// double and rounded once, cot = r e^-lv / n (or NULL); lv = logvar[b]
int launch_variance_loss(const float* x, const float* noise, const float* sigma, float sigma_data, const float* f, const float* logvar, float* loss,
                         float* cot, float* dlogvar, int B, int64_t n, cudaStream_t st);

// (cos, sin) table of the axial RoPE angles of QkRope with R = 4 nf: theta_j = (j < nf ? pos_y : pos_x)[t] * freqs[h, j], j < 2 nf
int launch_rope_table(const float* pos, const float* freqs, float2* out, int T_tokens, int nh, int nf, cudaStream_t st);

// dtype conversion helpers
int launch_f32_to_bf16(const float* in, bf16* out, int64_t n, cudaStream_t st);
template <typename T>
int launch_to_f32(const T* in, float* out, int64_t n, cudaStream_t st);

}  // namespace kdb
