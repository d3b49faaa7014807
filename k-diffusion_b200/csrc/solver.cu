// solver.cu -- HBM-bound elementwise kernels of the Karras ODE/SDE solver loop, the Karras
// preconditioner for opaque inner models, and counter-based noise (Philox normal fill, virtual
// Brownian tree).  All latents are fp32.  Every kernel moves 128 bits per load/store, four
// independent loads in flight per thread, grid sized to a multiple of the SM count.
//
// Reference semantics: k_diffusion/sampling.py:46-62 (to_d, ancestral step, default noise),
// :65-114 (Brownian noise), :117-184 (euler / euler_ancestral / heun), :584-607 (dpmpp_2m),
// k_diffusion/layers.py:70-74,88-90 (Denoiser scalings), k_diffusion/external.py:9-38,87-177 (external model wrappers).
#include <cmath>
#include <cstdarg>
#include <cstring>
#include <atomic>
#include <vector>

#include <cuda_fp16.h>

#include "common.cuh"

namespace kdb {

// ------------------------------------------------------------------------------------------------
// error + launch bookkeeping (shared by all translation units)
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches[F_COUNT];
static const char* kFamilyNames[F_COUNT] = {
    "solver", "precond", "noise", "patch_in", "patch_out", "cond", "rmsnorm", "gemm_simt", "gemm_tc",
    "qknorm_rope", "attn_generic", "attn_tc", "geglu", "merge_gather", "convert", "fused_norm",
    "unet_conv", "unet_adagn", "unet_resample", "unet_patch", "unet_cond", "unet_conv_tf32", "unet_attn_tf32",
    "unet_conv_fp16", "unet_attn_fp16", "mmd_tiles", "mmd_reduce", "poly_kernel", "col_mean", "cov",
    "gemm_tf32", "wgrad_tf32", "ema"};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (int)e;
}

// optional per-launch event trace (kdb_profile_begin / kdb_profile_end): an event after every launch;
// consecutive differences are per-kernel device times on a serialised stream.
static std::vector<cudaEvent_t> g_prof_events;
static std::vector<int> g_prof_family;
static bool g_prof_on = false;
static size_t g_prof_cap = 0;

void count_launch(int family, cudaStream_t st) {
  g_launches[family].fetch_add(1, std::memory_order_relaxed);
  if (g_prof_on && g_prof_family.size() < g_prof_cap) {
    cudaEvent_t ev = g_prof_events[g_prof_family.size() + 1];
    cudaEventRecord(ev, st);
    g_prof_family.push_back(family);
  }
}

// ------------------------------------------------------------------------------------------------
// elementwise engine
// ------------------------------------------------------------------------------------------------
enum EwOp { OP_EULER = 0, OP_EULER_NOISE, OP_HEUN2, OP_DPMPP2M, OP_DPMPP2M_1, OP_LINCOMB, OP_CFG };

struct EwParams {
  const float* in[6];
  float* out;
  float c[6];
  int n_in;
  int64_t n;
};

template <int OP>
__device__ __forceinline__ float ew_apply(const EwParams& p, const float (&v)[6]) {
  if constexpr (OP == OP_EULER) {                 // x + (x - den) * r
    return v[0] + (v[0] - v[1]) * p.c[0];
  } else if constexpr (OP == OP_EULER_NOISE) {    // x + (x - den) * r + noise * cn
    return (v[0] + (v[0] - v[1]) * p.c[0]) + v[2] * p.c[1];
  } else if constexpr (OP == OP_HEUN2) {          // x + ((x - den1) * a1 + (x2 - den2) * a2)
    return v[0] + ((v[0] - v[1]) * p.c[0] + (v[2] - v[3]) * p.c[1]);
  } else if constexpr (OP == OP_DPMPP2M) {        // a x - b (k1 den + k0 old)
    return p.c[0] * v[0] - p.c[1] * (p.c[2] * v[1] + p.c[3] * v[2]);
  } else if constexpr (OP == OP_DPMPP2M_1) {      // a x - b den
    return p.c[0] * v[0] - p.c[1] * v[1];
  } else if constexpr (OP == OP_CFG) {            // uncond + (cond - uncond) * scale  (reference train.py:341)
    return v[0] + (v[1] - v[0]) * p.c[0];
  } else {
    float acc = p.c[0] * v[0];
#pragma unroll
    for (int i = 1; i < 6; ++i)
      if (i < p.n_in) acc += p.c[i] * v[i];
    return acc;
  }
}

template <int OP> struct EwArity { static constexpr int value = 6; };
template <> struct EwArity<OP_EULER> { static constexpr int value = 2; };
template <> struct EwArity<OP_EULER_NOISE> { static constexpr int value = 3; };
template <> struct EwArity<OP_HEUN2> { static constexpr int value = 4; };
template <> struct EwArity<OP_DPMPP2M> { static constexpr int value = 3; };
template <> struct EwArity<OP_DPMPP2M_1> { static constexpr int value = 2; };
template <> struct EwArity<OP_CFG> { static constexpr int value = 2; };

constexpr int kEwThreads = 256;
constexpr int kEwUnroll = 4;

template <int OP, bool VEC>
__global__ void __launch_bounds__(kEwThreads) ew_kernel(const EwParams p) {
  constexpr int NIN = EwArity<OP>::value;
  const int n_in = (OP == OP_LINCOMB) ? p.n_in : NIN;
  if constexpr (VEC) {
    const int64_t n4 = p.n >> 2;
    const int64_t tile = (int64_t)kEwThreads * kEwUnroll;
    for (int64_t base = (int64_t)blockIdx.x * tile; base < n4; base += (int64_t)gridDim.x * tile) {
      float4 v[kEwUnroll][NIN];
#pragma unroll
      for (int u = 0; u < kEwUnroll; ++u) {
        const int64_t i = base + (int64_t)u * kEwThreads + threadIdx.x;
#pragma unroll
        for (int k = 0; k < NIN; ++k)
          if (k < n_in && i < n4) v[u][k] = __ldg(reinterpret_cast<const float4*>(p.in[k]) + i);
      }
#pragma unroll
      for (int u = 0; u < kEwUnroll; ++u) {
        const int64_t i = base + (int64_t)u * kEwThreads + threadIdx.x;
        if (i < n4) {
          float a[6], b[6], c[6], d[6];
#pragma unroll
          for (int k = 0; k < 6; ++k) {
            const bool on = k < NIN && k < n_in;
            a[k] = on ? v[u][k < NIN ? k : 0].x : 0.f;
            b[k] = on ? v[u][k < NIN ? k : 0].y : 0.f;
            c[k] = on ? v[u][k < NIN ? k : 0].z : 0.f;
            d[k] = on ? v[u][k < NIN ? k : 0].w : 0.f;
          }
          float4 o;
          o.x = ew_apply<OP>(p, a);
          o.y = ew_apply<OP>(p, b);
          o.z = ew_apply<OP>(p, c);
          o.w = ew_apply<OP>(p, d);
          reinterpret_cast<float4*>(p.out)[i] = o;
        }
      }
    }
    // tail (< 4 elements)
    const int64_t t0 = n4 << 2;
    if (blockIdx.x == 0 && threadIdx.x < (p.n - t0)) {
      const int64_t i = t0 + threadIdx.x;
      float a[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) a[k] = (k < NIN && k < n_in) ? p.in[k][i] : 0.f;
      p.out[i] = ew_apply<OP>(p, a);
    }
  } else {
    for (int64_t i = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * kEwThreads) {
      float a[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) a[k] = (k < NIN && k < n_in) ? p.in[k][i] : 0.f;
      p.out[i] = ew_apply<OP>(p, a);
    }
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int ew_grid(int64_t n, bool vec) {
  int64_t per_block = vec ? (int64_t)kEwThreads * kEwUnroll * 4 : kEwThreads;
  int64_t blocks = ceil_div(n, per_block);
  int64_t cap = (int64_t)kNumSMs * 8;           // 8 resident CTAs of 256 threads per SM
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

template <int OP>
static int ew_launch(const EwParams& p, int n_in, cudaStream_t st) {
  KDB_REQUIRE(p.n >= 0 && p.out != nullptr, KDB_ERR_BAD_ARG, "solver: bad n/out");
  if (p.n == 0) return 0;
  bool vec = aligned16(p.out);
  for (int k = 0; k < n_in; ++k) {
    KDB_REQUIRE(p.in[k] != nullptr, KDB_ERR_BAD_ARG, "solver: input %d is NULL", k);
    vec = vec && aligned16(p.in[k]);
  }
  if (vec)
    ew_kernel<OP, true><<<ew_grid(p.n, true), kEwThreads, 0, st>>>(p);
  else
    ew_kernel<OP, false><<<ew_grid(p.n, false), kEwThreads, 0, st>>>(p);
  KDB_LAUNCH_CHECK(F_SOLVER, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Karras preconditioner around an opaque inner model
// ------------------------------------------------------------------------------------------------
template <int MODE>   // 0: x*c_in   1: f*c_out + x*c_skip   2: (x - f)/sigma   3: (x + f*sigma)*c_in (f: the noise of a training loss)
__global__ void __launch_bounds__(256) precond_kernel(const float* __restrict__ f, const float* __restrict__ x,
                                                      const float* __restrict__ sigma, float sd, float* __restrict__ out,
                                                      int64_t per_sample, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int b = (int)(i / per_sample);
    if constexpr (MODE == 2) {
      out[i] = (x[i] - f[i]) / sigma[b];
    } else {
      float c_skip, c_out, c_in;
      karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
      if constexpr (MODE == 1)
        out[i] = f[i] * c_out + x[i] * c_skip;
      else if constexpr (MODE == 3)
        out[i] = __fmul_rn(__fadd_rn(x[i], __fmul_rn(f[i], sigma[b])), c_in);
      else
        out[i] = x[i] * c_in;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// External model wrappers (reference external.py:9-38, 87-177): scale-in and the eps / v combine around a foreign inner model.
// torch evaluates the reference's expressions one rounded operation per kernel, so every product, sum, square root and
// reciprocal here is an explicitly rounded intrinsic in the same order (nvcc would otherwise contract a*b + c into an FMA):
//   s2 = sigma * sigma + sd^2        c_in = rcp(sqrt(s2))           (`1 / t` is reciprocal(t) * 1 in torch)
//   eps: out = f * (-sigma) + x      v: out = f * c_out + x * c_skip, c_out = (-sigma * sd) / sqrt(s2), c_skip = rcp(s2) * sd^2
// As out = f * cf + x * cx (cx = 1 for eps: x * 1 is exact), one kernel serves scale-in (no f), both combines and, with either
// term dropped, their derivatives.
// ------------------------------------------------------------------------------------------------
enum ExtMode { EXT_SCALE_IN = 0, EXT_EPS = 1, EXT_V = 2 };

__device__ __forceinline__ void external_coefs(int mode, float sigma, float sd, float& cf, float& cx) {
  const float sd2 = __fmul_rn(sd, sd);
  const float s2 = __fadd_rn(__fmul_rn(sigma, sigma), sd2);
  if (mode == EXT_EPS) {
    cf = -sigma;
    cx = 1.f;
  } else if (mode == EXT_V) {
    cf = __fdiv_rn(__fmul_rn(-sigma, sd), __fsqrt_rn(s2));
    cx = __fmul_rn(__frcp_rn(s2), sd2);
  } else {
    cf = 0.f;
    cx = __frcp_rn(__fsqrt_rn(s2));
  }
}

__device__ __forceinline__ float ext_f(float v) { return v; }
__device__ __forceinline__ float ext_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float ext_f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float4 ext_load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
template <typename T>
__device__ __forceinline__ float4 ext_load4(const T* p) {         // four 16-bit values in one 8-byte load
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const T* h = reinterpret_cast<const T*>(&u);
  return make_float4(ext_f(h[0]), ext_f(h[1]), ext_f(h[2]), ext_f(h[3]));
}

__device__ __forceinline__ float ext_apply(bool has_f, bool has_x, float f, float x, float cf, float cx) {
  if (!has_f) return __fmul_rn(x, cx);
  if (!has_x) return __fmul_rn(f, cf);
  return __fadd_rn(__fmul_rn(f, cf), __fmul_rn(x, cx));
}

// blockIdx.y walks the samples (the per-sample coefficients are computed once per thread and sample), blockIdx.x the elements
// of one sample: 4 per thread and step when VEC (per_sample, f's batch stride and every pointer allow 128-bit x / out access).
template <typename TF, bool VEC>
__global__ void __launch_bounds__(256) external_kernel(int mode, const TF* f, int64_t f_stride, const float* x,
                                                       const float* __restrict__ sigma, float sd, float* out, int batch,
                                                       int64_t per_sample) {
  const bool has_f = f != nullptr, has_x = x != nullptr;
  for (int b = blockIdx.y; b < batch; b += gridDim.y) {
    float cf, cx;
    external_coefs(mode, __ldg(sigma + b), sd, cf, cx);
    const TF* fb = has_f ? f + (int64_t)b * f_stride : nullptr;
    const float* xb = has_x ? x + (int64_t)b * per_sample : nullptr;
    float* ob = out + (int64_t)b * per_sample;
    if constexpr (VEC) {
      for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < per_sample / 4; i += (int64_t)gridDim.x * 256) {
        const float4 fv = has_f ? ext_load4(fb + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 xv = has_x ? reinterpret_cast<const float4*>(xb)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        reinterpret_cast<float4*>(ob)[i] = make_float4(ext_apply(has_f, has_x, fv.x, xv.x, cf, cx), ext_apply(has_f, has_x, fv.y, xv.y, cf, cx),
                                                       ext_apply(has_f, has_x, fv.z, xv.z, cf, cx), ext_apply(has_f, has_x, fv.w, xv.w, cf, cx));
      }
    } else {
      for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < per_sample; i += (int64_t)gridDim.x * 256)
        ob[i] = ext_apply(has_f, has_x, has_f ? ext_f(fb[i]) : 0.f, has_x ? xb[i] : 0.f, cf, cx);
    }
  }
}

template <typename TF>
static int external_launch(int mode, const TF* f, int64_t f_stride, const float* x, const float* sigma, float sd, float* out, int batch,
                           int64_t per_sample, cudaStream_t st) {
  const auto al = [](const void* p, uintptr_t a) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
  const bool vec = per_sample % 4 == 0 && f_stride % 4 == 0 && al(f, 4 * sizeof(TF)) && al(x, 16) && al(out, 16);
  const int gy = batch < 65535 ? batch : 65535;
  int64_t gx = ceil_div(vec ? per_sample / 4 : per_sample, 256);
  const int64_t cap = (int64_t)kNumSMs * 8 / gy;                 // ~8 resident CTAs per SM over the whole grid
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  const dim3 grid((unsigned)gx, (unsigned)gy);
  if (vec)
    external_kernel<TF, true><<<grid, 256, 0, st>>>(mode, f, f_stride, x, sigma, sd, out, batch, per_sample);
  else
    external_kernel<TF, false><<<grid, 256, 0, st>>>(mode, f, f_stride, x, sigma, sd, out, batch, per_sample);
  KDB_LAUNCH_CHECK(F_PRECOND, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based normals
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}

__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f) + (1.0f / 33554432.0f); }

__device__ __forceinline__ float4 normal4(uint4 r) {
  float4 z;
  const float r0 = sqrtf(-2.0f * logf(u01(r.x)));
  const float r1 = sqrtf(-2.0f * logf(u01(r.z)));
  float s, c;
  sincospif(2.0f * u01(r.y), &s, &c);
  z.x = r0 * c;
  z.y = r0 * s;
  sincospif(2.0f * u01(r.w), &s, &c);
  z.z = r1 * c;
  z.w = r1 * s;
  return z;
}

constexpr uint32_t kTagNormal = 0x6e6f726du;    // "norm"
constexpr uint32_t kTagBrownian = 0x62726f77u;  // "brow"

__global__ void __launch_bounds__(256) noise_normal_kernel(float* __restrict__ out, const int64_t* __restrict__ seeds,
                                                           uint64_t stream_id, int64_t per_sample, int64_t groups_per_sample,
                                                           int64_t total_groups) {
  for (int64_t gi = (int64_t)blockIdx.x * 256 + threadIdx.x; gi < total_groups; gi += (int64_t)gridDim.x * 256) {
    const int64_t b = gi / groups_per_sample, g = gi - b * groups_per_sample;
    const uint64_t seed = (uint64_t)seeds[b];
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)stream_id, (uint32_t)(stream_id >> 32) ^ kTagNormal),
                                  make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float4 z = normal4(r);
    float* o = out + b * per_sample + g * 4;
    const int64_t left = per_sample - g * 4;
    if (left >= 4 && ((reinterpret_cast<uintptr_t>(o) & 15u) == 0)) {
      *reinterpret_cast<float4*>(o) = z;
    } else {
      const float zz[4] = {z.x, z.y, z.z, z.w};
      for (int j = 0; j < 4 && j < left; ++j) o[j] = zz[j];
    }
  }
}

// Box-Muller on the MUFU unit (lg2, sqrt, sin, cos: ~8 MUFU + 12 FP32 instructions for four normals instead of ~150 with the
// accurate logf / sincospif): the Brownian tree draws 25-50 of these per output group.  Absolute error, measured on an H100 80GB HBM3
// against float64 Box-Muller of the same uniforms (tests/test_gpu_noise.py): 1.4e-6 at the largest radius (u = 2^-25, r = 5.9), but
// 1.2e-4 at u = 1 - 2^-23, where r is only 4.9e-4 and the absolute error of __log2f near 1 (2^-22 in the CUDA guide) dominates; the
// guide's bounds allow up to 5.8e-4 there.  u = 1.0f gives exactly 0.
__device__ __forceinline__ float4 normal4_fast(uint4 r) {
  constexpr float kNeg2Ln2 = -1.3862943611198906f, kTwoPi = 6.283185307179586f;
  const float r0 = __fsqrt_rn(kNeg2Ln2 * __log2f(u01(r.x)));
  const float r1 = __fsqrt_rn(kNeg2Ln2 * __log2f(u01(r.z)));
  const float a0 = kTwoPi * (u01(r.y) - 0.5f), a1 = kTwoPi * (u01(r.w) - 0.5f);      // angle in (-pi, pi): no range reduction needed
  float4 z;
  z.x = r0 * __cosf(a0);
  z.y = r0 * __sinf(a0);
  z.z = r1 * __cosf(a1);
  z.w = r1 * __sinf(a1);
  return z;
}

// The virtual Brownian tree: W(t_min) = 0, W(t_max) ~ N(0, t_max - t_min), every dyadic midpoint is a Brownian bridge draw keyed by
// (seed, element group, node id); W(t) = `depth` bridge levels + linear interpolation inside the last interval.
struct BrownianWalk {
  double a, b;
  float4 wa, wb;
  uint32_t node;
};
__device__ __forceinline__ float4 brownian_mid(const BrownianWalk& w, uint2 key, uint32_t g_lo, uint32_t g_hi) {
  const float4 z = normal4_fast(philox4x32_10(make_uint4(g_lo, g_hi, w.node + 0x80000000u, kTagBrownian), key));
  const float sd = (float)(0.5 * sqrt(w.b - w.a));   // bridge std at the midpoint: sqrt((b-a)/4)
  return make_float4(fmaf(sd, z.x, 0.5f * (w.wa.x + w.wb.x)), fmaf(sd, z.y, 0.5f * (w.wa.y + w.wb.y)), fmaf(sd, z.z, 0.5f * (w.wa.z + w.wb.z)),
                     fmaf(sd, z.w, 0.5f * (w.wa.w + w.wb.w)));
}
__device__ __forceinline__ void brownian_step(BrownianWalk& w, double t, const float4 wm) {
  const double mid = 0.5 * (w.a + w.b);
  if (t < mid) { w.b = mid; w.wb = wm; w.node = w.node * 2u; }
  else { w.a = mid; w.wa = wm; w.node = w.node * 2u + 1u; }
}
__device__ __forceinline__ float4 brownian_finish(const BrownianWalk& w, double t) {
  const float f = (w.b > w.a) ? (float)((t - w.a) / (w.b - w.a)) : 0.f;
  return make_float4(fmaf(f, w.wb.x - w.wa.x, w.wa.x), fmaf(f, w.wb.y - w.wa.y, w.wa.y), fmaf(f, w.wb.z - w.wa.z, w.wa.z), fmaf(f, w.wb.w - w.wa.w, w.wa.w));
}

// out = (W(t1) - W(t0)) * inv_norm.  The two root-to-leaf walks share every level above the one where t0 and t1 fall on different
// sides of a midpoint (t0, t1 are kernel arguments: the branch is uniform), so the common prefix is drawn once.
__global__ void __launch_bounds__(256) noise_brownian_kernel(float* __restrict__ out, const int64_t* __restrict__ seeds,
                                                             int64_t per_sample, int64_t groups_per_sample, int64_t total_groups,
                                                             double t_min, double t_max, double t0, double t1, int depth, float inv_norm) {
  t0 = fmin(fmax(t0, t_min), t_max);
  t1 = fmin(fmax(t1, t_min), t_max);
  // level at which the walks part (host-free: recomputed per thread from the same scalars, ~depth double compares)
  int split = depth;
  {
    double a = t_min, b = t_max;
    for (int l = 0; l < depth; ++l) {
      const double mid = 0.5 * (a + b);
      if ((t0 < mid) != (t1 < mid)) { split = l; break; }
      if (t0 < mid) b = mid; else a = mid;
    }
  }
  const float sT = (float)sqrt(t_max - t_min);
  for (int64_t gi = (int64_t)blockIdx.x * 256 + threadIdx.x; gi < total_groups; gi += (int64_t)gridDim.x * 256) {
    const int64_t b = gi / groups_per_sample, g = gi - b * groups_per_sample;
    const uint64_t seed = (uint64_t)seeds[b];
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint32_t g_lo = (uint32_t)g, g_hi = (uint32_t)(g >> 32);
    const float4 zT = normal4_fast(philox4x32_10(make_uint4(g_lo, g_hi, 1u, kTagBrownian), key));
    BrownianWalk w0{t_min, t_max, make_float4(0.f, 0.f, 0.f, 0.f), make_float4(sT * zT.x, sT * zT.y, sT * zT.z, sT * zT.w), 1u};
    for (int l = 0; l < split; ++l) brownian_step(w0, t0, brownian_mid(w0, key, g_lo, g_hi));
    BrownianWalk w1 = w0;
    if (split < depth) {
      const float4 wm = brownian_mid(w0, key, g_lo, g_hi);        // the node where the walks part: one draw, two directions
      brownian_step(w0, t0, wm);
      brownian_step(w1, t1, wm);
      for (int l = split + 1; l < depth; ++l) {
        brownian_step(w0, t0, brownian_mid(w0, key, g_lo, g_hi));
        brownian_step(w1, t1, brownian_mid(w1, key, g_lo, g_hi));
      }
    }
    const float4 v0 = brownian_finish(w0, t0), v1 = brownian_finish(w1, t1);
    const float zz[4] = {(v1.x - v0.x) * inv_norm, (v1.y - v0.y) * inv_norm, (v1.z - v0.z) * inv_norm, (v1.w - v0.w) * inv_norm};
    float* o = out + b * per_sample + g * 4;
    const int64_t left = per_sample - g * 4;
    if (left >= 4 && ((reinterpret_cast<uintptr_t>(o) & 15u) == 0)) {
      *reinterpret_cast<float4*>(o) = make_float4(zz[0], zz[1], zz[2], zz[3]);
    } else {
      for (int j = 0; j < 4 && j < left; ++j) o[j] = zz[j];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// error norm of the adaptive DPM-Solver (sampling.py:466-468): sum over the latent of ((lo - hi) / max(atol, rtol max(|lo|, |prev|)))^2.
// Deterministic two-stage reduction: each CTA writes one partial (fixed grid, fixed order inside the CTA), the last stage adds the
// partials in index order.  partials[0] = result, partials[1 + b] = CTA b.
// ------------------------------------------------------------------------------------------------
constexpr int kErrBlocks = 296, kErrThreads = 256;

// RK = false: the DPM-Solver form above (a = lo, b = hi, c = prev).
// RK = true : the embedded Runge-Kutta form of the likelihood ODE (sampling.py:298, dopri5): a = error estimate, b = y0, c = y1,
//             sum (a / (atol + rtol max(|b|, |c|)))^2.
template <bool RK>
__global__ void __launch_bounds__(kErrThreads) dpm_error_partial_kernel(const float* __restrict__ lo, const float* __restrict__ hi,
                                                                        const float* __restrict__ prev, int64_t n, float atol, float rtol,
                                                                        float* __restrict__ partials) {
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * kErrThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kErrThreads) {
    const float a = __ldg(lo + i), b = __ldg(hi + i), c = __ldg(prev + i);
    float v;
    if constexpr (RK) {
      v = a / (atol + rtol * fmaxf(fabsf(b), fabsf(c)));
    } else {
      const float delta = fmaxf(atol, rtol * fmaxf(fabsf(a), fabsf(c)));
      v = (a - b) / delta;
    }
    acc = fmaf(v, v, acc);
  }
  __shared__ float red[kErrThreads];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kErrThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partials[1 + blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(32) dpm_error_final_kernel(float* __restrict__ partials, int blocks) {
  if (threadIdx.x == 0) {
    double acc = 0.0;
    for (int b = 0; b < blocks; ++b) acc += (double)partials[1 + b];
    partials[0] = (float)acc;
  }
}

}  // namespace kdb

using namespace kdb;

extern "C" {

int kdb_abi_version(void) { return KDB_ABI_VERSION; }
const char* kdb_last_error(void) { return g_err; }

uint64_t kdb_launch_count(void) {
  uint64_t t = 0;
  for (int i = 0; i < F_COUNT; ++i) t += g_launches[i].load(std::memory_order_relaxed);
  return t;
}

int kdb_launch_breakdown(const char** names, uint64_t* counts, int cap) {
  for (int i = 0; i < F_COUNT && i < cap; ++i) {
    if (names) names[i] = kFamilyNames[i];
    if (counts) counts[i] = g_launches[i].load(std::memory_order_relaxed);
  }
  return F_COUNT;
}

int kdb_profile_begin(int max_launches, void* stream) {
  KDB_REQUIRE(max_launches > 0 && !g_prof_on, KDB_ERR_BAD_ARG, "profile_begin: bad capacity or already profiling");
  while (g_prof_events.size() < (size_t)max_launches + 1) {
    cudaEvent_t ev;
    KDB_CUDA(cudaEventCreate(&ev));
    g_prof_events.push_back(ev);
  }
  g_prof_family.clear();
  g_prof_cap = (size_t)max_launches;
  KDB_CUDA(cudaEventRecord(g_prof_events[0], (cudaStream_t)stream));
  g_prof_on = true;
  return 0;
}

__global__ void profile_gate_kernel(unsigned long long ns) {
  unsigned long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  do {
    __nanosleep(2000);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  } while (t - t0 < ns);
}

int kdb_profile_gate(int64_t nanoseconds, void* stream) {
  KDB_REQUIRE(nanoseconds >= 0 && nanoseconds <= 2000000000ll, KDB_ERR_BAD_ARG, "profile_gate: 0 <= nanoseconds <= 2e9");
  profile_gate_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned long long)nanoseconds);
  KDB_CUDA(cudaGetLastError());
  return 0;
}

int kdb_profile_end(int* families_host, float* ms_host, int cap) {
  KDB_REQUIRE(g_prof_on, KDB_ERR_BAD_ARG, "profile_end: not profiling");
  g_prof_on = false;
  const int n = (int)g_prof_family.size();
  if (n > 0) KDB_CUDA(cudaEventSynchronize(g_prof_events[n]));
  for (int i = 0; i < n && i < cap; ++i) {
    float ms = 0.f;
    KDB_CUDA(cudaEventElapsedTime(&ms, g_prof_events[i], g_prof_events[i + 1]));
    if (families_host) families_host[i] = g_prof_family[i];
    if (ms_host) ms_host[i] = ms;
  }
  return n;
}

int kdb_solver_euler_step(const float* x, const float* den, const float* noise, float* x_out, int64_t n, float r, float cn,
                          void* stream) {
  EwParams p{};
  p.in[0] = x; p.in[1] = den; p.in[2] = noise; p.out = x_out; p.c[0] = r; p.c[1] = cn; p.n = n;
  if (noise) return ew_launch<OP_EULER_NOISE>(p, 3, (cudaStream_t)stream);
  return ew_launch<OP_EULER>(p, 2, (cudaStream_t)stream);
}

int kdb_solver_cfg_combine(const float* uncond, const float* cond, float* out, int64_t n, float scale, void* stream) {
  EwParams p{};
  p.in[0] = uncond; p.in[1] = cond; p.out = out; p.c[0] = scale; p.n = n;
  return ew_launch<OP_CFG>(p, 2, (cudaStream_t)stream);
}

int kdb_solver_dpm_error(const float* x_low, const float* x_high, const float* x_prev, int64_t n, float atol, float rtol, float* partials,
                         void* stream) {
  KDB_REQUIRE(x_low && x_high && x_prev && partials && n > 0, KDB_ERR_BAD_ARG, "dpm_error: bad args");
  dpm_error_partial_kernel<false><<<kErrBlocks, kErrThreads, 0, (cudaStream_t)stream>>>(x_low, x_high, x_prev, n, atol, rtol, partials);
  KDB_LAUNCH_CHECK(F_SOLVER, (cudaStream_t)stream);
  dpm_error_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(partials, kErrBlocks);
  KDB_LAUNCH_CHECK(F_SOLVER, (cudaStream_t)stream);
  return 0;
}

int kdb_solver_rk_error(const float* err, const float* y0, const float* y1, int64_t n, float atol, float rtol, float* partials,
                        void* stream) {
  KDB_REQUIRE(err && y0 && y1 && partials && n > 0, KDB_ERR_BAD_ARG, "rk_error: bad args");
  dpm_error_partial_kernel<true><<<kErrBlocks, kErrThreads, 0, (cudaStream_t)stream>>>(err, y0, y1, n, atol, rtol, partials);
  KDB_LAUNCH_CHECK(F_SOLVER, (cudaStream_t)stream);
  dpm_error_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(partials, kErrBlocks);
  KDB_LAUNCH_CHECK(F_SOLVER, (cudaStream_t)stream);
  return 0;
}

int kdb_solver_heun_correct(const float* x, const float* den1, const float* x2, const float* den2, float* x_out, int64_t n,
                            float a1, float a2, void* stream) {
  EwParams p{};
  p.in[0] = x; p.in[1] = den1; p.in[2] = x2; p.in[3] = den2; p.out = x_out; p.c[0] = a1; p.c[1] = a2; p.n = n;
  return ew_launch<OP_HEUN2>(p, 4, (cudaStream_t)stream);
}

int kdb_solver_dpmpp_2m_step(const float* x, const float* den, const float* old_den, float* x_out, int64_t n, float a, float b,
                             float k1, float k0, void* stream) {
  EwParams p{};
  p.in[0] = x; p.in[1] = den; p.in[2] = old_den; p.out = x_out; p.n = n;
  p.c[0] = a; p.c[1] = b; p.c[2] = k1; p.c[3] = k0;
  if (old_den == nullptr) {
    KDB_REQUIRE(k0 == 0.f && k1 == 1.f, KDB_ERR_BAD_ARG, "dpmpp_2m: old_den NULL requires k1=1,k0=0");
    return ew_launch<OP_DPMPP2M_1>(p, 2, (cudaStream_t)stream);
  }
  return ew_launch<OP_DPMPP2M>(p, 3, (cudaStream_t)stream);
}

int kdb_solver_lincomb(const float* const* in_host, const float* coef_host, int n_in, float* out, int64_t n, void* stream) {
  KDB_REQUIRE(n_in >= 1 && n_in <= 6 && in_host && coef_host, KDB_ERR_BAD_ARG, "lincomb: 1 <= n_in <= 6");
  EwParams p{};
  for (int i = 0; i < n_in; ++i) { p.in[i] = in_host[i]; p.c[i] = coef_host[i]; }
  p.out = out; p.n = n; p.n_in = n_in;
  return ew_launch<OP_LINCOMB>(p, n_in, (cudaStream_t)stream);
}

static int precond_grid(int64_t total) {
  int64_t blocks = ceil_div(total, 256);
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  return (int)(blocks < 1 ? 1 : blocks);
}

int kdb_solver_to_d(const float* x, const float* den, const float* sigma, float* out, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE(x && den && sigma && out && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "to_d: bad args");
  const int64_t total = (int64_t)batch * per_sample;
  precond_kernel<2><<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(den, x, sigma, 0.f, out, per_sample, total);
  KDB_LAUNCH_CHECK(F_SOLVER, (cudaStream_t)stream);
  return 0;
}

int kdb_precond_scale_in(const float* x, const float* sigma, float sigma_data, float* out, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE(x && sigma && out && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "precond_scale_in: bad args");
  const int64_t total = (int64_t)batch * per_sample;
  precond_kernel<0><<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(nullptr, x, sigma, sigma_data, out, per_sample, total);
  KDB_LAUNCH_CHECK(F_PRECOND, (cudaStream_t)stream);
  return 0;
}

int kdb_precond_combine(const float* f, const float* x, const float* sigma, float sigma_data, float* out, int batch,
                        int64_t per_sample, void* stream) {
  KDB_REQUIRE(f && x && sigma && out && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "precond_combine: bad args");
  const int64_t total = (int64_t)batch * per_sample;
  precond_kernel<1><<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(f, x, sigma, sigma_data, out, per_sample, total);
  KDB_LAUNCH_CHECK(F_PRECOND, (cudaStream_t)stream);
  return 0;
}

// The training losses of layers.py:76-86 (Denoiser, scales == 1) and :107-111 (SimpleLossDenoiser), one CTA per sample.  Each
// product and sum is rounded on its own, in the order of the reference's expressions; the mean is a fixed-order block sum.
__global__ void __launch_bounds__(256) denoiser_loss_kernel(int kind, const float* __restrict__ x, const float* __restrict__ noise,
                                                            const float* __restrict__ sigma, const float* __restrict__ weight, float sd,
                                                            const float* __restrict__ f, float* __restrict__ loss, float* __restrict__ cot,
                                                            int64_t per_sample) {
  __shared__ float red[8];
  const int64_t b = blockIdx.x;
  const float s = sigma[b];
  float c_skip, c_out, c_in;
  karras_scalings(s, sd, c_skip, c_out, c_in);
  const float w = kind == KDB_LOSS_DENOISER ? weight[b] : 1.f;
  const float inv_n = 1.f / (float)per_sample;
  // d loss / d f = 2 r g / N with r the residual: g = w (Denoiser), -c_out / sigma (SimpleLossDenoiser: r = eps - noise)
  const float g = kind == KDB_LOSS_DENOISER ? w : __fdiv_rn(-c_out, s);
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < per_sample; i += 256) {
    const int64_t j = b * per_sample + i;
    const float xn = __fadd_rn(x[j], __fmul_rn(noise[j], s));
    float r;
    if (kind == KDB_LOSS_DENOISER) {
      r = __fsub_rn(f[j], __fdiv_rn(__fsub_rn(x[j], __fmul_rn(c_skip, xn)), c_out));
    } else {
      const float den = __fadd_rn(__fmul_rn(f[j], c_out), __fmul_rn(xn, c_skip));
      r = __fsub_rn(__fdiv_rn(__fsub_rn(xn, den), s), noise[j]);
    }
    acc = __fadd_rn(acc, __fmul_rn(r, r));
    if (cot != nullptr) cot[j] = __fmul_rn(__fmul_rn(2.f * g, r), inv_n);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) loss[b] = __fmul_rn(__fdiv_rn(acc, (float)per_sample), w);
}

int kdb_loss_noised_input(const float* x, const float* noise, const float* sigma, float sigma_data, float* out, int batch, int64_t per_sample,
                          void* stream) {
  KDB_REQUIRE(x && noise && sigma && out && batch > 0 && per_sample > 0 && sigma_data > 0.f, KDB_ERR_BAD_ARG, "loss_noised_input: bad args");
  const int64_t total = (int64_t)batch * per_sample;
  precond_kernel<3><<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(noise, x, sigma, sigma_data, out, per_sample, total);
  KDB_LAUNCH_CHECK(F_PRECOND, (cudaStream_t)stream);
  return 0;
}

int kdb_denoiser_loss(int kind, const float* x, const float* noise, const float* sigma, const float* weight, float sigma_data, const float* f,
                      float* loss, float* cotangent, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE(x && noise && sigma && f && loss && batch > 0 && per_sample > 0 && sigma_data > 0.f, KDB_ERR_BAD_ARG, "denoiser_loss: bad args");
  KDB_REQUIRE(kind == KDB_LOSS_SIMPLE || (kind == KDB_LOSS_DENOISER && weight), KDB_ERR_BAD_ARG, "denoiser_loss: bad kind %d or NULL weight", kind);
  denoiser_loss_kernel<<<(unsigned)batch, 256, 0, (cudaStream_t)stream>>>(kind, x, noise, sigma, weight, sigma_data, f, loss, cotangent, per_sample);
  KDB_LAUNCH_CHECK(F_PRECOND, (cudaStream_t)stream);
  return 0;
}

int kdb_external_scale_in(const float* x, const float* sigma, float sigma_data, float* out, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE(x && sigma && out && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "external_scale_in: bad args");
  return external_launch<float>(EXT_SCALE_IN, nullptr, 0, x, sigma, sigma_data, out, batch, per_sample, (cudaStream_t)stream);
}

int kdb_external_combine(int kind, const void* f, int f_dtype, int64_t f_batch_stride, const float* x, const float* sigma, float sigma_data,
                         float* out, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE((f || x) && sigma && out && batch > 0 && per_sample > 0 && f_batch_stride >= 0, KDB_ERR_BAD_ARG,
              "external_combine: bad args (f and x may not both be NULL)");
  KDB_REQUIRE(kind == KDB_EXTERNAL_EPS || kind == KDB_EXTERNAL_V, KDB_ERR_BAD_ARG, "external_combine: kind %d is neither eps nor v", kind);
  const int mode = kind == KDB_EXTERNAL_EPS ? EXT_EPS : EXT_V;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (f_dtype) {
    case KDB_DTYPE_F32:
      return external_launch(mode, static_cast<const float*>(f), f_batch_stride, x, sigma, sigma_data, out, batch, per_sample, st);
    case KDB_DTYPE_F16:
      return external_launch(mode, static_cast<const __half*>(f), f_batch_stride, x, sigma, sigma_data, out, batch, per_sample, st);
    case KDB_DTYPE_BF16:
      return external_launch(mode, static_cast<const bf16*>(f), f_batch_stride, x, sigma, sigma_data, out, batch, per_sample, st);
    default:
      set_error("external_combine: f_dtype %d is not KDB_DTYPE_F32 / F16 / BF16", f_dtype);
      return KDB_ERR_BAD_ARG;
  }
}

int kdb_noise_normal(float* out, const int64_t* seeds, uint64_t stream_id, int batch, int64_t per_sample, void* stream) {
  KDB_REQUIRE(out && seeds && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "noise_normal: bad args");
  const int64_t gps = ceil_div(per_sample, 4), total = gps * batch;
  noise_normal_kernel<<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(out, seeds, stream_id, per_sample, gps, total);
  KDB_LAUNCH_CHECK(F_NOISE, (cudaStream_t)stream);
  return 0;
}

int kdb_noise_brownian(float* out, const int64_t* seeds, int batch, int64_t per_sample, double t_min, double t_max, double t0,
                       double t1, int depth, void* stream) {
  KDB_REQUIRE(out && seeds && batch > 0 && per_sample > 0, KDB_ERR_BAD_ARG, "noise_brownian: bad args");
  KDB_REQUIRE(t_max > t_min && depth >= 1 && depth <= 30, KDB_ERR_BAD_ARG, "noise_brownian: need t_max > t_min, 1 <= depth <= 30");
  KDB_REQUIRE(t0 != t1, KDB_ERR_BAD_ARG, "noise_brownian: t0 == t1");
  const int64_t gps = ceil_div(per_sample, 4), total = gps * batch;
  const float inv_norm = (float)(1.0 / std::sqrt(std::fabs(t1 - t0)));
  noise_brownian_kernel<<<precond_grid(total), 256, 0, (cudaStream_t)stream>>>(out, seeds, per_sample, gps, total, t_min, t_max, t0, t1,
                                                                              depth, inv_norm);
  KDB_LAUNCH_CHECK(F_NOISE, (cudaStream_t)stream);
  return 0;
}

}  // extern "C"
