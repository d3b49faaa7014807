// common.cuh -- shared helpers for libkdb200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>

#include "kdiffusion_b200.h"

namespace kdb {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

// launch accounting (kdb_launch_count / kdb_launch_breakdown)
enum Family {
  F_SOLVER = 0, F_PRECOND, F_NOISE, F_PATCH_IN, F_PATCH_OUT, F_COND, F_RMSNORM, F_GEMM_SIMT, F_GEMM_TC,
  F_QKNORM_ROPE, F_ATTN_GENERIC, F_ATTN_TC, F_GEGLU, F_MERGE_GATHER, F_CONVERT, F_FUSED_NORM,
  F_UNET_CONV, F_UNET_ADAGN, F_UNET_RESAMPLE, F_UNET_PATCH, F_UNET_COND, F_UNET_CONV_TF32, F_UNET_ATTN_TF32,
  F_UNET_CONV_FP16, F_UNET_ATTN_FP16, F_MMD_TILES, F_MMD_REDUCE, F_POLY_KERNEL, F_COL_MEAN, F_COV,
  F_GEMM_TF32, F_WGRAD_TF32, F_EMA, F_AUGMENT, F_COUNT
};
void count_launch(int family, cudaStream_t st);

#define KDB_LAUNCH_CHECK(fam, st)                                    \
  do {                                                               \
    ::kdb::count_launch(fam, st);                                    \
    cudaError_t e__ = cudaGetLastError();                            \
    if (e__ != cudaSuccess) return ::kdb::cuda_fail(e__, #fam);      \
  } while (0)

#define KDB_CUDA(call)                                               \
  do {                                                               \
    cudaError_t e__ = (call);                                        \
    if (e__ != cudaSuccess) return ::kdb::cuda_fail(e__, #call);     \
  } while (0)

#define KDB_REQUIRE(cond, code, ...)                                 \
  do {                                                               \
    if (!(cond)) { ::kdb::set_error(__VA_ARGS__); return (code); }   \
  } while (0)

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// sum of v over the CTA, in the same order on every thread; red: shared scratch of one float per warp
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += red[i];
  return t;
}

constexpr float kRsqrt2 = 0.70710678118654752440f;
// erf GELU (image_transformer_v2.py:89-95, layers.py of image_v1) in the reference's association, 0.5 g (1 + erf(g / sqrt 2))
__device__ __forceinline__ float gelu_erf(float g) { return 0.5f * g * (1.f + erff(g * kRsqrt2)); }

// torch.lerp(self, end, w) in fp32 as ATen computes it (ATen/native/Lerp.h): |w| < 0.5 ? self + w (end - self) : end - (end - self) (1 - w),
// each branch one fused multiply-add as nvcc contracts it in torch's kernel, written with explicit roundings so that no contraction here
// can change it.  The TokenSplit lerps and the EMA update share it.
__device__ __forceinline__ float lerp_torch(float self, float end, float w) {
  const float d = __fsub_rn(end, self);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, d, self) : __fmaf_rn(-d, __fsub_rn(1.f, w), end);
}

// Karras preconditioner scalings (reference layers.py:70-74), fp32 like the reference.
__device__ __forceinline__ void karras_scalings(float sigma, float sd, float& c_skip, float& c_out, float& c_in) {
  float s2 = sigma * sigma + sd * sd;
  float rs = sqrtf(s2);
  c_skip = sd * sd / s2;
  c_out = sigma * sd / rs;
  c_in = 1.0f / rs;
}

// Patch addressing: token tok of a [B, th, tw] token grid is token (ty, tx) of image b; pixel (y, x) of channel c of image b sits
// at nchw_offset in an NCHW [B, C, H, W] image.
__device__ __forceinline__ void token_coords(int64_t tok, int th, int tw, int& b, int& ty, int& tx) {
  const int64_t per = (int64_t)th * tw;
  b = (int)(tok / per);
  const int r = (int)(tok - (int64_t)b * per);
  ty = r / tw;
  tx = r - ty * tw;
}
__device__ __forceinline__ int64_t nchw_offset(int b, int c, int y, int x, int C, int H, int W) {
  return (((int64_t)b * C + c) * H + y) * W + x;
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

constexpr int kNumSMs = 132;   // H100 SXM; the launchers query the device where it matters

// Opens `kernel` to `bytes` of dynamic shared memory on its first launch (flag: one static per kernel).
template <typename K>
int set_smem_once(K kernel, bool& flag, int bytes) {
  if (!flag) {
    KDB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    flag = true;
  }
  return 0;
}

}  // namespace kdb

// Programmatic dependent launch: let the CTAs of the next kernel in the stream (if it was launched with the programmatic
// attribute -- attention and the fused feed-forward kernel are) be scheduled as soon as every CTA of this grid has passed this point or exited.
// The caller must itself be past any dependency on ITS predecessor, i.e. ordinary (fully serialised) launches call it first thing.
#define KDB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")

