// patch_kernels.cu -- tiled patch-in / patch-out kernels: persistent CTAs, weights staged once in shared memory, 64-token
// tiles, register-tiled fp32 FMA (each thread owns a tokens x outputs micro-tile fed by 128-bit shared loads), coalesced
// pixel and token I/O.
//   patch_in : x[B,C,H,W] * c_in(sigma) -> 'b (h nh) (w nw) c -> b h w (nh nw c)' -> Linear(K=ph*pw*C -> N)
//              (reference image_transformer_v2.py:586-595,723-724 and layers.py:88-90 for c_in)
//   patch_out: RMSNorm(out_norm) -> Linear(C0 -> ph*pw*Cout) -> 'b h w (nh nw c) -> b c (h nh) (w nw)' -> c_out*F + c_skip*x
//              (reference :598-607,758-760 and layers.py:88-90)
// Both are <0.5 % of the model's MACs; their job is to stay close to the HBM bound (25 MB in / 17-34 MB out at B=32).
#include <algorithm>

#include "model_kernels.cuh"

namespace kdb {
namespace {

constexpr int TOK = 64;
constexpr float kEps = 1e-6f;

struct PatchGeom {
  int C, H, W, th, tw;   // image channels / size, token grid
  int64_t tokens;
};

// coordinates of token (tile origin + t) from the tile origin's coordinates, without 64-bit division
__device__ __forceinline__ void tok_step(const PatchGeom& g, int b0, int ty0, int tx0, int t, int& b, int& ty, int& tx) {
  b = b0; ty = ty0; tx = tx0 + t;
  while (tx >= g.tw) { tx -= g.tw; ++ty; }
  while (ty >= g.th) { ty -= g.th; ++b; }
}

template <typename T> __device__ __forceinline__ void store8(T* o, const float (&a)[8]);
template <> __device__ __forceinline__ void store8<float>(float* o, const float (&a)[8]) {
  reinterpret_cast<float4*>(o)[0] = make_float4(a[0], a[1], a[2], a[3]);
  reinterpret_cast<float4*>(o)[1] = make_float4(a[4], a[5], a[6], a[7]);
}
template <> __device__ __forceinline__ void store8<bf16>(bf16* o, const float (&a)[8]) {
  __nv_bfloat162 h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a[2 * i], a[2 * i + 1]);
  *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(h);
}

// ------------------------------------------------------------------------------------------------
// patch_in: thread = TT tokens x 8 outputs, TT = N / 32 (N = 64, 128, 256)
// ------------------------------------------------------------------------------------------------
template <typename T, int PH, int PW, int TT>
__global__ void __launch_bounds__(256) patch_in_tiled(const float* __restrict__ x, const float* __restrict__ sigma, float sd,
                                                      const float* __restrict__ W, T* __restrict__ out, PatchGeom g) {
  KDB_PDL_TRIGGER();
  extern __shared__ __align__(16) float sm[];
  constexpr int N = TT * 32;
  const int K = PH * PW * g.C;
  float* patch = sm;                 // [K][TOK]
  float* Ws = sm + K * TOK;          // [K][N]
  for (int idx = threadIdx.x; idx < K * N; idx += 256) {   // W [N][K] -> Ws [K][N], once per CTA
    const int n = idx / K, k = idx - n * K;
    Ws[k * N + n] = __ldg(W + idx);
  }
  const int ng = threadIdx.x % (N / 8), tg = threadIdx.x / (N / 8);    // output group (8 wide), token group (TT wide)
  const int64_t n_tiles = (g.tokens + TOK - 1) / TOK;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t tok0 = tile * TOK;
    int b0, ty0, tx0;
    token_coords(tok0, g.th, g.tw, b0, ty0, tx0);
    __syncthreads();                      // previous tile's patch fully consumed (and Ws visible on the first pass)
    // gather pixels, pixel-contiguous order: idx = ((c*PH + nh)*TOK + t)*PW + nw.  All loads of a thread are issued
    // before any is consumed (the kernel is latency-bound otherwise).
    constexpr int GI = 16;                                   // K*TOK/256 <= 16 (K <= 64)
    float gv[GI];
#pragma unroll
    for (int it = 0; it < GI; ++it) {
      const int idx = threadIdx.x + it * 256;
      gv[it] = 0.f;
      if (idx < K * TOK) {
        const int nw = idx % PW;
        const int t = (idx / PW) % TOK;
        const int rest = idx / (PW * TOK);
        const int nh = rest % PH, c = rest / PH;
        if (tok0 + t < g.tokens) {
          int b, ty, tx;
          tok_step(g, b0, ty0, tx0, t, b, ty, tx);
          gv[it] = __ldg(x + nchw_offset(b, c, ty * PH + nh, tx * PW + nw, g.C, g.H, g.W));
        }
      }
    }
#pragma unroll
    for (int it = 0; it < GI; ++it) {
      const int idx = threadIdx.x + it * 256;
      if (idx < K * TOK) {
        const int nw = idx % PW;
        const int t = (idx / PW) % TOK;
        const int rest = idx / (PW * TOK);
        const int nh = rest % PH, c = rest / PH;
        float c_in = 1.f;
        if (sd > 0.f && tok0 + t < g.tokens) {
          int b, ty, tx;
          tok_step(g, b0, ty0, tx0, t, b, ty, tx);
          c_in = rsqrtf(fmaf(__ldg(sigma + b), __ldg(sigma + b), sd * sd));
        }
        patch[((nh * PW + nw) * g.C + c) * TOK + t] = gv[it] * c_in;
      }
    }
    __syncthreads();
    float acc[TT][8];
#pragma unroll
    for (int i = 0; i < TT; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int k = 0; k < K; ++k) {
      const float4 w0 = *reinterpret_cast<const float4*>(Ws + k * N + ng * 8), w1 = *reinterpret_cast<const float4*>(Ws + k * N + ng * 8 + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      float a[TT];
      if constexpr (TT % 4 == 0) {
#pragma unroll
        for (int i = 0; i < TT; i += 4) {
          const float4 p4 = *reinterpret_cast<const float4*>(patch + k * TOK + tg * TT + i);
          a[i] = p4.x; a[i + 1] = p4.y; a[i + 2] = p4.z; a[i + 3] = p4.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < TT; ++i) a[i] = patch[k * TOK + tg * TT + i];
      }
#pragma unroll
      for (int i = 0; i < TT; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < TT; ++i) {
      const int64_t tok = tok0 + tg * TT + i;
      if (tok < g.tokens) store8<T>(out + tok * N + ng * 8, acc[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// patch_out: thread = 4 tokens x 4 outputs (N = ph*pw*Cout <= 64, N % 4 == 0)
// ------------------------------------------------------------------------------------------------
template <typename T, int PH, int PW>
__global__ void __launch_bounds__(256) patch_out_tiled(const T* __restrict__ tokens, const float* __restrict__ nscale,
                                                       const float* __restrict__ W, const float* __restrict__ x_in,
                                                       const float* __restrict__ sigma, float sd, float* __restrict__ out, PatchGeom g,
                                                       int C0) {
  extern __shared__ __align__(16) float sm[];
  const int Cout = g.C;
  const int N = PH * PW * Cout;
  constexpr int XS = TOK + 4;                       // row stride of xn / ys (keeps 16-byte alignment, skews banks)
  float* xn = sm;                                   // [C0][XS]
  float* Ws = xn + C0 * XS;                         // [C0][N]
  float* ys = Ws + C0 * N;                          // [N][XS]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int idx = threadIdx.x; idx < N * C0; idx += 256) {      // W [N][C0] -> Ws [C0][N], once per CTA
    const int n = idx / C0, k = idx - n * C0;
    Ws[k * N + n] = __ldg(W + idx);
  }
  const int ngroups = N / 4;
  const int og = threadIdx.x % ngroups, tg = threadIdx.x / ngroups;      // 4 outputs, 4 tokens (tg < 16)
  const int64_t n_tiles = (g.tokens + TOK - 1) / TOK;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t tok0 = tile * TOK;
    int b0, ty0, tx0;
    token_coords(tok0, g.th, g.tw, b0, ty0, tx0);
    __syncthreads();                       // previous tile's xn / ys consumed
    // RMSNorm: warp per token (8 tokens per warp), normalised row written transposed.  For C0 <= 256 the 8 rows are
    // fetched into registers up front (8 x C0/32 independent loads per lane) so the loads overlap.
    if (C0 <= 256) {
      float rv[8][8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t tok = tok0 + warp + 8 * j;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = lane + 32 * i;
          rv[j][i] = (tok < g.tokens && c < C0) ? to_f(tokens[tok * C0 + c]) : 0.f;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) ss = fmaf(rv[j][i], rv[j][i], ss);
        ss = warp_sum(ss);
        const float rstd = rsqrtf(ss / (float)C0 + kEps);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = lane + 32 * i;
          if (c < C0) xn[c * XS + warp + 8 * j] = to_f(from_f<T>(rv[j][i] * (__ldg(nscale + c) * rstd)));
        }
      }
    } else {
      for (int t = warp; t < TOK; t += 8) {
        const int64_t tok = tok0 + t;
        float ss = 0.f;
        if (tok < g.tokens)
          for (int c = lane; c < C0; c += 32) {
            const float v = to_f(tokens[tok * C0 + c]);
            ss = fmaf(v, v, ss);
          }
        ss = warp_sum(ss);
        const float rstd = rsqrtf(ss / (float)C0 + kEps);
        for (int c = lane; c < C0; c += 32) {
          const float v = tok < g.tokens ? to_f(tokens[tok * C0 + c]) : 0.f;
          xn[c * XS + t] = to_f(from_f<T>(v * (__ldg(nscale + c) * rstd)));
        }
      }
    }
    __syncthreads();
    if (tg < TOK / 4) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      for (int k = 0; k < C0; ++k) {
        const float4 a4 = *reinterpret_cast<const float4*>(xn + k * XS + tg * 4);
        const float4 w4 = *reinterpret_cast<const float4*>(Ws + k * N + og * 4);
        const float a[4] = {a4.x, a4.y, a4.z, a4.w}, w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<float4*>(ys + (og * 4 + j) * XS + tg * 4) =
            make_float4(to_f(from_f<T>(acc[0][j])), to_f(from_f<T>(acc[1][j])), to_f(from_f<T>(acc[2][j])), to_f(from_f<T>(acc[3][j])));
    }
    __syncthreads();
    // scatter in pixel-contiguous order: idx = ((c*PH + nh)*TOK + t)*PW + nw; x_in loads batched ahead of their use
    constexpr int SI = 16;                                   // N*TOK/256 <= 16 (N <= 64)
    float xv[SI];
    int64_t ov[SI];
#pragma unroll
    for (int it = 0; it < SI; ++it) {
      const int idx = threadIdx.x + it * 256;
      ov[it] = -1;
      xv[it] = 0.f;
      if (idx < N * TOK) {
        const int nw = idx % PW;
        const int tt = (idx / PW) % TOK;
        const int rest = idx / (PW * TOK);
        const int nh = rest % PH, c = rest / PH;
        if (tok0 + tt < g.tokens) {
          int b, ty, tx;
          tok_step(g, b0, ty0, tx0, tt, b, ty, tx);
          ov[it] = nchw_offset(b, c, ty * PH + nh, tx * PW + nw, Cout, g.H, g.W);
          if (sd > 0.f) xv[it] = __ldg(x_in + ov[it]);
        }
      }
    }
#pragma unroll
    for (int it = 0; it < SI; ++it) {
      const int idx = threadIdx.x + it * 256;
      if (ov[it] >= 0) {
        const int nw = idx % PW;
        const int tt = (idx / PW) % TOK;
        const int rest = idx / (PW * TOK);
        const int nh = rest % PH, c = rest / PH;
        const float y = ys[((nh * PW + nw) * Cout + c) * XS + tt];
        if (sd > 0.f) {
          int b, ty, tx;
          tok_step(g, b0, ty0, tx0, tt, b, ty, tx);
          float c_skip, c_out, c_in;
          karras_scalings(__ldg(sigma + b), sd, c_skip, c_out, c_in);
          out[ov[it]] = y * c_out + xv[it] * c_skip;
        } else {
          out[ov[it]] = y;
        }
      }
    }
  }
}

constexpr int kSmemMax = 160 * 1024;

template <typename T, int PH, int PW, int TT>
int run_patch_in(const float* x, const float* sigma, float sd, const float* W, T* out, const PatchGeom& g, size_t smem, cudaStream_t st) {
  static bool attr = false;
  int rc = set_smem_once(patch_in_tiled<T, PH, PW, TT>, attr, kSmemMax);
  if (rc) return rc;
  patch_in_tiled<T, PH, PW, TT><<<(unsigned)std::min<int64_t>(ceil_div(g.tokens, TOK), kNumSMs * 2), 256, smem, st>>>(x, sigma, sd, W, out, g);
  KDB_LAUNCH_CHECK(F_PATCH_IN, st);
  return 0;
}

template <typename T, int PH, int PW>
int run_patch_out(const T* tokens, const float* ns, const float* W, const float* x_in, const float* sigma, float sd, float* out,
                  const PatchGeom& g, int C0, size_t smem, cudaStream_t st) {
  static bool attr = false;
  int rc = set_smem_once(patch_out_tiled<T, PH, PW>, attr, kSmemMax);
  if (rc) return rc;
  patch_out_tiled<T, PH, PW><<<(unsigned)std::min<int64_t>(ceil_div(g.tokens, TOK), kNumSMs * 2), 256, smem, st>>>(tokens, ns, W, x_in, sigma, sd,
                                                                                                                  out, g, C0);
  KDB_LAUNCH_CHECK(F_PATCH_OUT, st);
  return 0;
}

}  // namespace

template <typename T>
bool launch_patch_in_tiled(const float* x, const float* sigma, float sigma_data, const float* W, T* out, int B, int C, int H, int Wd, int ph,
                           int pw, int N, cudaStream_t st, int* rc) {
  const int K = ph * pw * C;
  const size_t smem = sizeof(float) * ((size_t)K * TOK + (size_t)K * N);
  if (smem > kSmemMax || (N != 64 && N != 128 && N != 256) || !((ph == 4 && pw == 4) || (ph == 2 && pw == 2))) return false;
  PatchGeom g{C, H, Wd, H / ph, Wd / pw, (int64_t)B * (H / ph) * (Wd / pw)};
#define KDB_PI(PH_, PW_)                                                                                   \
  switch (N) {                                                                                             \
    case 64: *rc = run_patch_in<T, PH_, PW_, 2>(x, sigma, sigma_data, W, out, g, smem, st); return true;   \
    case 128: *rc = run_patch_in<T, PH_, PW_, 4>(x, sigma, sigma_data, W, out, g, smem, st); return true;  \
    default: *rc = run_patch_in<T, PH_, PW_, 8>(x, sigma, sigma_data, W, out, g, smem, st); return true;   \
  }
  if (ph == 4) { KDB_PI(4, 4) }
  KDB_PI(2, 2)
#undef KDB_PI
}
template bool launch_patch_in_tiled<float>(const float*, const float*, float, const float*, float*, int, int, int, int, int, int, int, cudaStream_t, int*);
template bool launch_patch_in_tiled<bf16>(const float*, const float*, float, const float*, bf16*, int, int, int, int, int, int, int, cudaStream_t, int*);

template <typename T>
bool launch_patch_out_tiled(const T* tokens, const float* norm_scale, const float* W, const float* x_in, const float* sigma, float sigma_data,
                            float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st, int* rc) {
  const int N = ph * pw * Cout;
  const size_t smem = sizeof(float) * ((size_t)C0 * (TOK + 4) + (size_t)C0 * N + (size_t)N * (TOK + 4));
  if (N > 64 || N % 4 != 0 || smem > kSmemMax || !((ph == 4 && pw == 4) || (ph == 2 && pw == 2))) return false;
  PatchGeom g{Cout, H, Wd, H / ph, Wd / pw, (int64_t)B * (H / ph) * (Wd / pw)};
  if (ph == 4)
    *rc = run_patch_out<T, 4, 4>(tokens, norm_scale, W, x_in, sigma, sigma_data, out, g, C0, smem, st);
  else
    *rc = run_patch_out<T, 2, 2>(tokens, norm_scale, W, x_in, sigma, sigma_data, out, g, C0, smem, st);
  return true;
}
template bool launch_patch_out_tiled<float>(const float*, const float*, const float*, const float*, const float*, float, float*, int, int, int,
                                            int, int, int, int, cudaStream_t, int*);
template bool launch_patch_out_tiled<bf16>(const bf16*, const float*, const float*, const float*, const float*, float, float*, int, int, int,
                                           int, int, int, int, cudaStream_t, int*);

}  // namespace kdb
