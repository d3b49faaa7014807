// tc_kernels.cuh -- wgmma / TMA kernels for the bf16 fast path (sm_90a).
#pragma once
#include "model_kernels.cuh"

namespace kdb {

// C[M,N] = A[M,K] W[N,K]^T (+ epilogue), bf16 operands staged by TMA, fp32 accumulators in registers (wgmma).
bool tc_gemm_supported(int64_t M, int N, int K, const GemmEpi& epi);
// Fused RMSNorm: a RESID / SPLIT_LERP GEMM with N % 128 == 0 can leave sum(x^2) of every row it writes ([rows, SS_PARTS] fp32, one slot per 128
// channels) and a STORE / QKV_ROPE / GEGLU GEMM whose A operand is that x can apply 1/rms in its epilogue (GemmEpi::ss_out / ss_in).
constexpr int SS_PARTS = 8;
bool tc_gemm_emits_rowss(int64_t M, int N, int K, const GemmEpi& epi);
int launch_gemm_tc(const bf16* A, const bf16* W, bf16* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st);

// up_proj with the GEGLU fused into the epilogue; W rows interleaved 8 value / 8 gate (engine.cu).
bool tc_gemm_geglu_supported(int64_t M, int N2, int K, bool fused_norm = false);
int launch_gemm_tc_geglu(const bf16* A, const bf16* W_il, bf16* out, int64_t M, int N2, int K, cudaStream_t st, const float* ss_in = nullptr);

// The whole feed-forward block of a 128-wide level in one kernel (tc_ffn_fused.cuh): x <- x + down(value(x_n) * gelu(gate(x_n))), in place.
// w_up_il carries the AdaRMSNorm channel scale (fold kernel) and the value / gate row interleave; ss_in = row statistics of x (required),
// ss_out = where to leave sum(x_new^2) per row (or nullptr).  KDB200_NO_FFN_FUSE=1 disables it (the two stand-alone GEMMs run instead).
bool tc_ffn_fused_supported(int64_t M, int C, int dff);
int launch_ffn_fused(bf16* x, const bf16* w_up_il, const bf16* w_down, int64_t M, int C, int dff, const float* ss_in, float* ss_out, cudaStream_t st);

// W'[n,k] = W[n,k] * g[k] for a table of weight matrices (AdaRMSNorm channel scale folded into the consumer weights)
struct FoldDesc {
  const bf16* src;
  bf16* dst;
  int rows, K, ada_off;
};
int launch_fold_norm_weights(const FoldDesc* descs_dev, int n_desc, const float* cond_row, cudaStream_t st);

// patch_out (4x4 patches, 3 channels): xn bf16 [M, C0] x W_pad bf16 [64, C0] -> fp32 NCHW with the Karras combine fused.
// ss_in != nullptr: xn is the RAW residual stream, W_pad carries out_norm.scale and the epilogue applies 1/rms per token.
bool tc_patch_out_supported(int C0, int Cout, int ph, int pw, int Wimg);
int launch_patch_out_tc(const bf16* xn, const bf16* W_pad, const float* x_in, const float* sigma, float sigma_data, float* out, int B, int H,
                        int Wimg, int C0, cudaStream_t st, const float* ss_in = nullptr);

// patch_in (4x4 patches of a 3-channel fp32 latent) on the tensor core; W_perm = prepare_patch_in_weight(patch_in.proj.weight)
bool tc_patch_in_supported(int Cin, int ph, int pw, int C0, int Wimg);
int prepare_patch_in_weight(const float* W, bf16* out_perm, int C0, cudaStream_t st);
int launch_patch_in_tc(const float* x, const float* sigma, float sigma_data, const bf16* W_perm, bf16* out, int B, int H, int Wimg, int C0,
                       float* ss_out, cudaStream_t st);

bool tc_attention_supported(int h, int w, int nh, int e, int attn_type, int attn_param);
// logit_bound: [nh] device floats with |q . k| <= bound per head (the layer's cosine-similarity scale), or nullptr.  With a bound the
// kernels use it as softmax's fixed shift (single pass, no row maximum); the caller guarantees bound <= KDB_ATTN_MAX_BOUND.
constexpr float KDB_ATTN_MAX_BOUND = 40.f;
int launch_attention_tc(const bf16* qkv, bf16* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                        cudaStream_t st, const float* logit_bound = nullptr);

template <typename T>
inline int attention_dispatch(const T* qkv, T* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                              cudaStream_t st, const float* logit_bound = nullptr) {
  (void)logit_bound;
  return launch_attention_generic<T>(qkv, out, B, h, w, nh, e, attn_type, attn_param, shift, st);
}
template <>
inline int attention_dispatch<bf16>(const bf16* qkv, bf16* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param,
                                    int shift, cudaStream_t st, const float* logit_bound) {
  if (tc_attention_supported(h, w, nh, e, attn_type, attn_param))
    return launch_attention_tc(qkv, out, B, h, w, nh, e, attn_type, attn_param, shift, st, logit_bound);
  return launch_attention_generic<bf16>(qkv, out, B, h, w, nh, e, attn_type, attn_param, shift, st);
}

}  // namespace kdb
