// unet_kernels.cuh -- launchers of the fp32 image_v1 U-Net kernels (reference models/image_v1.py, layers.py:116-313).
// Activations are token-major: [B, H, W, C] fp32, channels contiguous (DESIGN.md section 3).  Every kernel is deterministic:
// fixed reduction orders, no atomics.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace kdb {

// out[m, n] = bias[n] + sum_{tap, c} w[n, tap, c] * in(pixel m shifted by tap, c) + resid[m, n]
// A ks x ks convolution (ks = 1 or 3, zero padding ks / 2, stride 1) run as an implicit GEMM.  The input is the channel
// concatenation of in1 [B,H,W,c1] and in2 [B,H,W,c2] (c2 = 0: one source), so a UBlock's torch.cat is never materialised.
// w is tap-major [N, ks*ks, c1 + c2]; bias and the residual may be NULL.  The residual is [B,H,W,N] read as the concatenation of
// r1 (rc1 channels) and r2 (N - rc1 channels).  c1, c2 and rc1 must be multiples of 4.
struct ConvArgs {
  const float* in1 = nullptr;
  const float* in2 = nullptr;
  int c1 = 0, c2 = 0;
  const float* w = nullptr;
  const float* bias = nullptr;
  const float* r1 = nullptr;
  const float* r2 = nullptr;
  int rc1 = 0;
  float* out = nullptr;
  int B = 0, H = 0, W = 0, N = 0;
};
int launch_unet_conv(const ConvArgs& a, int ks, cudaStream_t st);
// The same convolution on the tensor cores at KDB_PREC_TF32 (unet_tf32.cu): tf32 operands, fp32 accumulation.  w is expected rounded
// to tf32 (launch_unet_round_tf32); activations are truncated to tf32 by the MMA.
// family: the launch family it is counted under (kdb_launch_breakdown)
int launch_unet_conv_tf32(const ConvArgs& a, int ks, cudaStream_t st, int family = F_UNET_CONV_TF32);
// ... at KDB_PREC_FP16 (unet_tf32.cu): fp16 operands, fp32 accumulation.  a.w is not read: w is the fp16 tap-major weight
// [N, ks*ks, f16_weight_ld(c1 + c2)] (launch_unet_round_f16); activations are rounded to the nearest fp16 (ties to even) in registers.
// An operand of magnitude >= 65520 becomes +-inf (no saturation).
int launch_unet_conv_fp16(const ConvArgs& a, const __half* w, int ks, cudaStream_t st);
// the row length of an fp16 weight of `channels` input channels: rounded up to 8 (16-byte rows for TMA; the padding is never read)
int f16_weight_ld(int channels);
// Global self-attention at KDB_PREC_TF32 / KDB_PREC_FP16 (unet_tf32.cu): qkv [B, T, 3 nh 64] fp32 in (t nh e) order with 1/sqrt(d_head)
// folded into q -> out [B, T, nh 64] fp32; q, k, v and the softmax probabilities truncated to tf32 / rounded to fp16 (nearest even),
// fp32 scores, softmax and accumulation, running-maximum softmax.  Any T >= 1.  unet_attn_tc_supported: the head sizes they are built
// for (64); the engine keeps attn_generic for the others.
bool unet_attn_tc_supported(int d_head);
int launch_unet_attn_tf32(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st);
int launch_unet_attn_fp16(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st);
// dst[i] = src[i] rounded to the nearest tf32 value (ties away from zero), stored as fp32
int launch_unet_round_tf32(const float* src, float* dst, int64_t n, cudaStream_t st);
// src [rows, C] fp32 -> dst [rows, f16_weight_ld(C)] fp16, rounded to nearest even (+-inf past 65504), the padding zero
int launch_unet_round_f16(const float* src, __half* dst, int64_t rows, int C, cudaStream_t st);

// AdaGN (layers.py:172-175), optionally followed by the erf GELU: out = [gelu](group_norm(x) * (1 + weight) + bias) with the
// (weight, bias) pair read from the conditioning row of image b at cond + b * cond_bs + ada_off (C weights, then C biases).
// x is the concatenation of in1 (c1 channels) and in2 (c2 channels, may be 0); out is [B, HW, c1 + c2].  One CTA per
// (group, image) reduces the group's mean and variance in a fixed order, then normalises the group.
int launch_unet_adagn(const float* in1, int c1, const float* in2, int c2, float* out, const float* cond, int64_t cond_bs, int ada_off,
                      int groups, bool gelu, int B, int HW, cudaStream_t st);

// Downsample2d / Upsample2d (layers.py:251-280): depthwise [1,3,3,1]/8 filter, reflect padding 1, stride 2.
// in [B, H, W, C] -> out [B, H/2, W/2, C] (up = false) or [B, 2H, 2W, C] (up = true).  H, W >= 2.
int launch_unet_resample(const float* in, float* out, int B, int H, int W, int C, bool up, cudaStream_t st);

// pixel_unshuffle(c_in(sigma) x, p) then proj_in (1x1 conv with bias): x [B, Cin, H, W] NCHW -> out [B, H/p, W/p, N]
// (image_v1.py:146-148, layers.py:88-90).  sigma_data <= 0: no c_in scaling.  w [N, Cin*p*p].
int launch_unet_patch_in(const float* x, const float* sigma, float sigma_data, const float* w, const float* bias, float* out, int B, int Cin,
                         int H, int W, int p, int N, cudaStream_t st);

// proj_out (1x1 conv with bias) then pixel_shuffle, the variance channel (has_variance) skipped, then (sigma_data > 0) the
// Karras combine out = c_out F + c_skip x_in (image_v1.py:150-154, layers.py:88-90).  tokens [B, H/p, W/p, K], w [>= Cout*p*p, K],
// out [B, Cout, H, W] NCHW.
int launch_unet_patch_out(const float* tokens, const float* w, const float* bias, const float* x_in, const float* sigma, float sigma_data,
                          float* out, int B, int Cout, int H, int W, int p, int K, cudaStream_t st);

// Conditioning (image_v1.py:136-139, augmentation.py:97-104, and every AdaGN mapper, layers.py:173): per row
//   cond = MappingNet(FourierFeatures(log(sigma) / 4) + mapping_cond_linear(v)),  v = [aug_cond or zeros(9), mapping_cond] with the
//   augment wrapper, mapping_cond otherwise (NULL: no term);  out[row] = [ada_w cond + ada_b (ada_total floats), cond (mw floats)].
struct UNetCondWeights {
  int mw = 0, mcond_dim = 0, augment = 0, ada_total = 0;
  const float *time_emb = nullptr, *mcond_w = nullptr;
  const float *map_w0 = nullptr, *map_b0 = nullptr, *map_w1 = nullptr, *map_b1 = nullptr;
  const float *ada_w = nullptr, *ada_b = nullptr;   // [ada_total, mw], [ada_total]
};
int launch_unet_conditioning(const UNetCondWeights& w, int rows, const float* sigma, const float* aug, const float* mcond, float* out,
                             int64_t out_stride, cudaStream_t st);

// torch conv weight [N, C, k, k] -> tap-major [N, k*k, C], times `scale` for rows n < scaled_rows (the folded attention scale)
int launch_unet_reorder_conv_weight(const float* src, float* dst, int N, int C, int ks, int scaled_rows, float scale, cudaStream_t st);

}  // namespace kdb
