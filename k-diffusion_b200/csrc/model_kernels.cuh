// model_kernels.cuh -- launchers for the per-op kernels of the image_transformer_v2 forward pass.
// "generic" kernels are precision-templated SIMT kernels (fp32 = the exact path used for the
// rtol 1e-3 / atol 1e-5 parity gate; bf16 = fallback for shapes the tensor-core kernels do not cover).
#pragma once
#include "common.cuh"

namespace kdb {

enum GemmEpilogue { EPI_STORE = 0, EPI_RESID = 1, EPI_SPLIT_LERP = 2, EPI_QKV_ROPE = 3 };

struct GemmEpi {
  int mode = EPI_STORE;
  const void* resid = nullptr;   // EPI_RESID: [M,N] same type as out.  EPI_SPLIT_LERP: skip [B, 2hc, 2wc, C]
  const float* fac = nullptr;    // EPI_SPLIT_LERP: device scalar (TokenSplit.fac)
  int hc = 0, wc = 0, C = 0;     // EPI_SPLIT_LERP: coarse grid and fine channel count (N == 4*C)
  // EPI_QKV_ROPE (tensor-core path only): cosine-sim scaling + axial RoPE of the q and k thirds (N == 3*C, d_head 64)
  const float2* rope = nullptr;  // launch_rope_table: float4 [nh][8][T_tokens] = (cos, cos, sin, sin) of the angle pairs
  const float* qk_scale = nullptr;   // [nh]
  int nh = 0, T_tokens = 0;
  // TokenMerge folded into the A-operand load (tensor-core path only): A = fine tokens [B, 2*mhc, 2*mwc, mC], K = 4*mC in
  // (nh nw e) order, M = B*mhc*mwc.  mC == 0 -> A is a plain [M, K] matrix.
  int mhc = 0, mwc = 0, mC = 0;
  // fused RMSNorm (tensor-core kernel only).  Consumer (EPI_STORE / EPI_QKV_ROPE): A is the raw residual stream, W
  // already carries the channel scale, ss_in [M, 8] holds sum(x^2) per 128-channel block of every row and the epilogue scales
  // the accumulator by 1/rms (q/k thirds of EPI_QKV_ROPE are scale invariant).  Producer (EPI_RESID / EPI_SPLIT_LERP): ss_out
  // receives those sums for the rows written.
  const float* ss_in = nullptr;
  float* ss_out = nullptr;
};

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

// in-place cosine-sim scaling of q,k and axial RoPE on qkv [rows, 3, nh, e]  (image_transformer_v2.py:106-114,187-199,245-248)
// pos [T,2] (y,x) for the level, freqs [nh, e/8], scale [nh]; rows = B*T
template <typename T>
int launch_qknorm_rope(T* qkv, const float* pos, const float* freqs, const float* scale, int64_t rows, int T_tokens, int nh, int e,
                       cudaStream_t st);

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

// (cos, sin) table of the axial RoPE angles: out[t, h, j] for j < 2*nf: theta = (j < nf ? pos_y : pos_x)[t] * freqs[h, j % nf]
int launch_rope_table(const float* pos, const float* freqs, float2* out, int T_tokens, int nh, int nf, cudaStream_t st);

// dtype conversion helpers
int launch_f32_to_bf16(const float* in, bf16* out, int64_t n, cudaStream_t st);
template <typename T>
int launch_to_f32(const T* in, float* out, int64_t n, cudaStream_t st);

}  // namespace kdb
