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
  F_QKNORM_ROPE, F_ATTN_GENERIC, F_ATTN_TC, F_GEGLU, F_MERGE_GATHER, F_CONVERT, F_FUSED_NORM, F_COUNT
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

// Karras preconditioner scalings (reference layers.py:70-74), fp32 like the reference.
__device__ __forceinline__ void karras_scalings(float sigma, float sd, float& c_skip, float& c_out, float& c_in) {
  float s2 = sigma * sigma + sd * sd;
  float rs = sqrtf(s2);
  c_skip = sd * sd / s2;
  c_out = sigma * sd / rs;
  c_in = 1.0f / rs;
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

constexpr int kNumSMs = 132;   // H100 SXM; the launchers query the device where it matters

}  // namespace kdb

// Programmatic dependent launch: let the CTAs of the next kernel in the stream (if it was launched with the programmatic
// attribute -- attention and the fused feed-forward kernel are) be scheduled as soon as every CTA of this grid has passed this point or exited.
// The caller must itself be past any dependency on ITS predecessor, i.e. ordinary (fully serialised) launches call it first thing.
#define KDB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")

