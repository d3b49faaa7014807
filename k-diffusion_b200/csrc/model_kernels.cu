// model_kernels.cu -- precision-templated SIMT kernels for every op of the image_transformer_v2
// forward pass (reference: k_diffusion/models/image_transformer_v2.py).  With T = float this is the
// fp32-exact path behind the rtol 1e-3 / atol 1e-5 parity gate: all reductions accumulate in fp32,
// transcendental functions are the accurate (non fast-math) variants.  With T = bf16 the same
// kernels serve as the fallback for shapes the tensor-core (wgmma) kernels do not cover.
#include <algorithm>
#include <cmath>

#include "attn_sets.cuh"
#include "model_kernels.cuh"
#include "simt_tile.cuh"

namespace kdb {

constexpr float kEps = 1e-6f;   // RMSNorm / cosine-sim eps (image_transformer_v2.py:143,378)

// grid of a grid-stride kernel of 256 threads over n elements
static unsigned grid_stride_blocks(int64_t n) { return (unsigned)std::min<int64_t>(ceil_div(n, 256), kNumSMs * 16); }

// Tangent of a row norm y = x r, r = rsqrt(ss / n + eps), ss = sum x^2 (RMSNorm: n = row width; cosine-sim: n = 1, the layer's eps), along
// u with sd = x . u: dy = r u - x r^3 sd / n.  The row sums are the caller's.
struct NormTangent {
  float r, r3m;
  __device__ NormTangent(float ss, float sd, float n, float eps = kEps) : r(rsqrtf(ss / n + eps)), r3m(r * r * r * (sd / n)) {}
  __device__ float operator()(float x, float u) const { return r * u - x * r3m; }
};

// Axial RoPE of the first R columns of a head (QkRope): column j < R/2 pairs with column j + R/2 and both turn by
// theta_j = pos_y f_j (j < nf) or pos_x f_j (j >= nf), nf = R/4, f = the head's R/2 frequencies; columns from R on pass through.
__device__ __forceinline__ void rope_sincos(float py, float px, const float* f, int j, int nf, float& s, float& c) {
  sincosf((j < nf ? py : px) * f[j], &s, &c);
}
// column d of the rotated head v; INV: rotated by -theta (the transpose)
template <bool INV>
__device__ __forceinline__ float rope_rotate(const float* v, int d, int R, float py, float px, const float* f) {
  const int dr = R / 2;
  if (d >= R) return v[d];
  const int j = d < dr ? d : d - dr;
  float s, c;
  rope_sincos(py, px, f, j, R / 4, s, c);
  const float x1 = v[j], x2 = v[j + dr];
  if constexpr (INV)
    return d < dr ? x1 * c + x2 * s : x2 * c - x1 * s;
  else
    return d < dr ? x1 * c - x2 * s : x2 * c + x1 * s;
}

// the erf GELU's derivatives' form: gelu = g Phi(g) and slope = Phi(g) + g phi(g)
__device__ __forceinline__ void gelu_erf_slope(float g, float& gelu, float& slope) {
  const float Phi = 0.5f * (1.f + erff(g * kRsqrt2));
  const float phi = 0.39894228040143267794f * expf(-0.5f * g * g);
  gelu = g * Phi;
  slope = fmaf(g, phi, Phi);
}

// ------------------------------------------------------------------------------------------------
// patch_in: pixel-unshuffle + Linear (K = ph*pw*C is tiny: 16 or 48)
// ------------------------------------------------------------------------------------------------
constexpr int kPiTok = 8;

template <typename T>
__global__ void __launch_bounds__(128) patch_in_kernel(const float* __restrict__ x, const float* __restrict__ sigma, float sd,
                                                       const float* __restrict__ W, T* __restrict__ out, int C, int H, int Wd, int ph,
                                                       int pw, int N, int tw_n, int64_t tokens_total) {
  extern __shared__ float patch[];   // [kPiTok][K]
  const int K = ph * pw * C;
  const int th_n = H / ph;
  const int64_t tok0 = (int64_t)blockIdx.x * kPiTok;
  for (int idx = threadIdx.x; idx < kPiTok * K; idx += blockDim.x) {
    const int t = idx / K, k = idx - t * K;
    const int64_t tok = tok0 + t;
    float v = 0.f;
    if (tok < tokens_total) {
      int b, ty, tx;
      token_coords(tok, th_n, tw_n, b, ty, tx);
      float c_in = 1.f;
      if (sd > 0.f) {
        float cs, co;
        karras_scalings(sigma[b], sd, cs, co, c_in);
      }
      v = x[patch_pixel(b, ty, tx, k, C, H, Wd, ph, pw)] * c_in;
    }
    patch[idx] = v;
  }
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float acc[kPiTok];
#pragma unroll
    for (int t = 0; t < kPiTok; ++t) acc[t] = 0.f;
    const float* wr = W + (int64_t)n * K;
    for (int k = 0; k < K; ++k) {
      const float wv = __ldg(wr + k);
#pragma unroll
      for (int t = 0; t < kPiTok; ++t) acc[t] = fmaf(patch[t * K + k], wv, acc[t]);
    }
#pragma unroll
    for (int t = 0; t < kPiTok; ++t)
      if (tok0 + t < tokens_total) out[(tok0 + t) * N + n] = from_f<T>(acc[t]);
  }
}

template <typename T>
int launch_patch_in(const float* x, const float* sigma, float sigma_data, const float* W, T* out, int B, int C, int H, int Wd, int ph,
                    int pw, int N, cudaStream_t st) {
  KDB_REQUIRE(H % ph == 0 && Wd % pw == 0, KDB_ERR_BAD_SHAPE, "patch_in: %dx%d not divisible by patch %dx%d", H, Wd, ph, pw);
  {
    int rc = 0;
    if (launch_patch_in_tiled<T>(x, sigma, sigma_data, W, out, B, C, H, Wd, ph, pw, N, st, &rc)) return rc;
  }
  const int64_t tokens = (int64_t)B * (H / ph) * (Wd / pw);
  const int K = ph * pw * C;
  const size_t smem = sizeof(float) * kPiTok * K;
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "patch_in: patch too large (K=%d)", K);
  patch_in_kernel<T><<<(unsigned)ceil_div(tokens, kPiTok), 128, smem, st>>>(x, sigma, sigma_data, W, out, C, H, Wd, ph, pw, N, Wd / pw,
                                                                            tokens);
  KDB_LAUNCH_CHECK(F_PATCH_IN, st);
  return 0;
}
template int launch_patch_in<float>(const float*, const float*, float, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
template int launch_patch_in<bf16>(const float*, const float*, float, const float*, bf16*, int, int, int, int, int, int, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// RMSNorm with per-batch or shared scale: one warp per token row
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ scale,
                                                      int64_t scale_bstride, int64_t rows_per_batch, int64_t rows, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + row * C;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = to_f(xr[c]);
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)C + kEps);
  const float* sc = scale + (row / rows_per_batch) * scale_bstride;
  T* yr = y + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = from_f<T>(to_f(xr[c]) * (__ldg(sc + c) * rstd));
}

// bf16 fast variant: 16-byte loads/stores, G lanes per row (G = 16 or 32), CH chunks of 8 channels per lane, row kept in registers
template <int G, int CH>
__global__ void __launch_bounds__(256) rmsnorm_bf16_vec_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const float* __restrict__ scale,
                                                               int64_t scale_bstride, int64_t rows_per_batch, int64_t rows) {
  KDB_PDL_TRIGGER();
  constexpr int C = G * CH * 8;
  constexpr int ROWS_PER_WARP = 32 / G;
  const int lane = threadIdx.x & 31;
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t row = warp_id * ROWS_PER_WARP + lane / G;
  const int sub = lane % G;
  const bool live = row < rows;
  float v[CH][8];
  float ss = 0.f;
#pragma unroll
  for (int ch = 0; ch < CH; ++ch) {
    uint4 raw = make_uint4(0u, 0u, 0u, 0u);
    if (live) raw = __ldg(reinterpret_cast<const uint4*>(x + row * C + (sub + ch * G) * 8));
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[t]);
      v[ch][2 * t] = __low2float(h);
      v[ch][2 * t + 1] = __high2float(h);
      ss = fmaf(v[ch][2 * t], v[ch][2 * t], ss);
      ss = fmaf(v[ch][2 * t + 1], v[ch][2 * t + 1], ss);
    }
  }
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (!live) return;
  const float rstd = rsqrtf(ss / (float)C + kEps);
  const float* sc = scale + (row / rows_per_batch) * scale_bstride;
#pragma unroll
  for (int ch = 0; ch < CH; ++ch) {
    const int c0 = (sub + ch * G) * 8;
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(sc + c0)), s1 = __ldg(reinterpret_cast<const float4*>(sc + c0 + 4));
    const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(v[ch][2 * t] * (s[2 * t] * rstd), v[ch][2 * t + 1] * (s[2 * t + 1] * rstd));
      o[t] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(y + row * C + c0) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

template <typename T>
bool rmsnorm_fast(const T*, T*, const float*, int64_t, int64_t, int64_t, int, cudaStream_t) { return false; }
template <>
bool rmsnorm_fast<bf16>(const bf16* x, bf16* y, const float* scale, int64_t bs, int64_t rpb, int64_t rows, int C, cudaStream_t st) {
  if ((reinterpret_cast<uintptr_t>(scale) & 15) != 0 || (bs % 4) != 0) return false;
#define KDB_RMS(G_, CH_)                                                                                              \
  rmsnorm_bf16_vec_kernel<G_, CH_><<<(unsigned)ceil_div(rows, 8 * (32 / G_)), 256, 0, st>>>(x, y, scale, bs, rpb, rows); \
  return true;
  switch (C) {
    case 128: KDB_RMS(16, 1)
    case 256: KDB_RMS(32, 1)
    case 512: KDB_RMS(32, 2)
    case 768: KDB_RMS(32, 3)
    case 1024: KDB_RMS(32, 4)
    default: return false;
  }
#undef KDB_RMS
}

template <typename T>
int launch_rmsnorm(const T* x, T* y, const float* scale, int64_t scale_bstride, int64_t rows_per_batch, int64_t rows, int C,
                   cudaStream_t st) {
  if (rmsnorm_fast<T>(x, y, scale, scale_bstride, rows_per_batch, rows, C, st)) {
    KDB_LAUNCH_CHECK(F_RMSNORM, st);
    return 0;
  }
  rmsnorm_kernel<T><<<(unsigned)ceil_div(rows, 8), 256, 0, st>>>(x, y, scale, scale_bstride, rows_per_batch, rows, C);
  KDB_LAUNCH_CHECK(F_RMSNORM, st);
  return 0;
}
template int launch_rmsnorm<float>(const float*, float*, const float*, int64_t, int64_t, int64_t, int, cudaStream_t);
template int launch_rmsnorm<bf16>(const bf16*, bf16*, const float*, int64_t, int64_t, int64_t, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// SIMT GEMM, C = A W^T, fp32 accumulate, on the tile loop of simt_tile.cuh.
// ------------------------------------------------------------------------------------------------

template <typename T>
__device__ __forceinline__ void load4(const T* p, bool ok, float (&v)[4]);
template <>
__device__ __forceinline__ void load4<float>(const float* p, bool ok, float (&v)[4]) {
  if (ok) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else { v[0] = v[1] = v[2] = v[3] = 0.f; }
}
template <>
__device__ __forceinline__ void load4<bf16>(const bf16* p, bool ok, float (&v)[4]) {
  if (ok) {
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&t.x);
    const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&t.y);
    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
  } else { v[0] = v[1] = v[2] = v[3] = 0.f; }
}

template <typename T, typename TW, int EPI>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const T* __restrict__ A, const TW* __restrict__ W, T* __restrict__ Cout,
                                                        int64_t M, int N, int K, const T* __restrict__ resid,
                                                        const float* __restrict__ fac, int hc, int wc, int Cf) {
  const int64_t m0 = (int64_t)blockIdx.y * kTileM;
  const int n0 = blockIdx.x * kTileN;
  const int tid = threadIdx.x;
  const int lr = tid >> 2, lk = (tid & 3) * 4;   // loader: row 0..63, k offset 0,4,8,12
  auto fill = [&](int k0, TileSmem& As, TileSmem& Ws) {
    float av[4], wv[4];
    load4<T>(A + (m0 + lr) * K + k0 + lk, (m0 + lr) < M && (k0 + lk) < K, av);
    load4<TW>(W + (int64_t)(n0 + lr) * K + k0 + lk, (n0 + lr) < N && (k0 + lk) < K, wv);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[lk + i][lr] = av[i];
      Ws[lk + i][lr] = wv[i];
    }
  };
  simt_tile(m0, n0, M, N, K, fill, [&](int64_t m, int n, float acc) {
    if constexpr (EPI == EPI_STORE) {
      Cout[m * N + n] = from_f<T>(acc);
    } else if constexpr (EPI == EPI_RESID) {
      Cout[m * N + n] = from_f<T>(acc + to_f(resid[m * N + n]));
    } else {
      // TokenSplit: row m = (b, hy, wx) on the coarse grid, column n = (nh, nw, e)
      int b, hy, wx;
      token_coords(m, hc, wc, b, hy, wx);
      const int q = n / Cf, e = n - q * Cf;
      const int64_t dst = fine_offset(b, hy, wx, q, e, hc, wc, Cf);
      Cout[dst] = from_f<T>(lerp_torch(to_f(resid[dst]), acc, __ldg(fac)));
    }
  });
}

template <typename T, typename TW>
int launch_gemm_simt(const T* A, const TW* W, T* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st) {
  KDB_REQUIRE(K % 4 == 0, KDB_ERR_BAD_SHAPE, "gemm_simt: K=%d must be a multiple of 4", K);
  KDB_REQUIRE(M > 0 && N > 0, KDB_ERR_BAD_SHAPE, "gemm_simt: empty problem");
  dim3 grid((unsigned)ceil_div(N, kTileN), (unsigned)ceil_div(M, kTileM));
  KDB_REQUIRE(grid.y <= 65535u * 16u, KDB_ERR_BAD_SHAPE, "gemm_simt: M too large");
  if (grid.y > 65535u) {   // split M so gridDim.y stays legal
    const int64_t chunk = 65535LL * kTileM;
    for (int64_t mo = 0; mo < M; mo += chunk) {
      GemmEpi e2 = epi;
      KDB_REQUIRE(epi.mode != EPI_SPLIT_LERP, KDB_ERR_UNSUPPORTED, "gemm_simt: split-lerp with M > 4M rows");
      if (epi.mode == EPI_RESID) e2.resid = static_cast<const T*>(epi.resid) + mo * N;
      int rc = launch_gemm_simt<T, TW>(A + mo * K, W, C + mo * N, (M - mo) < chunk ? (M - mo) : chunk, N, K, e2, st);
      if (rc) return rc;
    }
    return 0;
  }
  const T* resid = static_cast<const T*>(epi.resid);
  switch (epi.mode) {
    case EPI_STORE:
      gemm_simt_kernel<T, TW, EPI_STORE><<<grid, 256, 0, st>>>(A, W, C, M, N, K, nullptr, nullptr, 0, 0, 0);
      break;
    case EPI_RESID:
      gemm_simt_kernel<T, TW, EPI_RESID><<<grid, 256, 0, st>>>(A, W, C, M, N, K, resid, nullptr, 0, 0, 0);
      break;
    case EPI_SPLIT_LERP:
      KDB_REQUIRE(N == 4 * epi.C && M % ((int64_t)epi.hc * epi.wc) == 0, KDB_ERR_BAD_SHAPE, "gemm_simt: bad split-lerp geometry");
      gemm_simt_kernel<T, TW, EPI_SPLIT_LERP><<<grid, 256, 0, st>>>(A, W, C, M, N, K, resid, epi.fac, epi.hc, epi.wc, epi.C);
      break;
    default:
      KDB_REQUIRE(false, KDB_ERR_BAD_ARG, "gemm_simt: bad epilogue %d", epi.mode);
  }
  KDB_LAUNCH_CHECK(F_GEMM_SIMT, st);
  return 0;
}
template int launch_gemm_simt<float, float>(const float*, const float*, float*, int64_t, int, int, const GemmEpi&, cudaStream_t);
template int launch_gemm_simt<bf16, bf16>(const bf16*, const bf16*, bf16*, int64_t, int, int, const GemmEpi&, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// cosine-sim scaling + axial RoPE of q and k from src to dst (src == dst: in place; else v is copied through).  One warp per (token row,
// head).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) qknorm_rope_kernel(const T* src, T* dst, const float* __restrict__ pos, const QkRope qr,
                                                          int64_t rows, int Ttok, int nh, int e) {
  extern __shared__ float sm[];   // [warps][2][e]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (item >= rows * nh) return;
  const int64_t row = item / nh;
  const int h = (int)(item - row * nh);
  float* buf = sm + (size_t)warp * 2 * e;
  const float py = pos[(row % Ttok) * 2 + 0], px = pos[(row % Ttok) * 2 + 1];
  const float sqs = sqrtf(qr.scale[h]);
  const float* f = qr.freqs + h * (qr.R / 2);
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int64_t off = (row * 3 + t) * (int64_t)nh * e + (int64_t)h * e;
    const T* v = src + off;
    float ss = 0.f;
    for (int d = lane; d < e; d += 32) {
      const float f = to_f(v[d]);
      ss = fmaf(f, f, ss);
    }
    ss = warp_sum(ss);
    const float sc = sqs * rsqrtf(ss + qr.eps);
    // the reference rounds the scaled q/k back to the activation dtype before RoPE (:114)
    for (int d = lane; d < e; d += 32) buf[t * e + d] = to_f(from_f<T>(to_f(v[d]) * sc));
    __syncwarp();
    for (int d = lane; d < e; d += 32) dst[off + d] = from_f<T>(rope_rotate<false>(buf + t * e, d, qr.R, py, px, f));
    __syncwarp();
  }
  if (src != dst) {
    const int64_t off = (row * 3 + 2) * (int64_t)nh * e + (int64_t)h * e;
    for (int d = lane; d < e; d += 32) dst[off + d] = src[off + d];
  }
}

static int check_qk_rope(const char* what, const QkRope& qr, int e) {
  KDB_REQUIRE(e % 8 == 0 && qr.R % 4 == 0 && qr.R > 0 && qr.R <= e, KDB_ERR_BAD_SHAPE,
              "%s: d_head %d must be a multiple of 8 and the rotated width %d a multiple of 4, at most d_head", what, e, qr.R);
  return 0;
}

template <typename T>
int launch_qknorm_rope(const T* src, T* dst, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e, cudaStream_t st) {
  if (int rc = check_qk_rope("qknorm_rope", qr, e)) return rc;
  const size_t smem = sizeof(float) * 4 * 2 * e;
  qknorm_rope_kernel<T><<<(unsigned)ceil_div(rows * nh, 4), 128, smem, st>>>(src, dst, pos, qr, rows, T_tokens, nh, e);
  KDB_LAUNCH_CHECK(F_QKNORM_ROPE, st);
  return 0;
}
template int launch_qknorm_rope<float>(const float*, float*, const float*, const QkRope&, int64_t, int, int, int, cudaStream_t);
template int launch_qknorm_rope<bf16>(const bf16*, bf16*, const float*, const QkRope&, int64_t, int, int, int, cudaStream_t);

// RoPE table for the QKV epilogue: float4 [(head * nf + i) * T + token] = (cos t_2i, cos t_2i+1, sin t_2i, sin t_2i+1), i < nf.
// Token-minor, so the 32 threads of an epilogue warp (32 consecutive tokens) read 512 contiguous bytes per load, and the
// (cos, cos, sin, sin) order is what the packed-fp32 rotation consumes.  theta_j = pos_h * f_j (j < nf) or pos_w * f_j (j >= nf),
// f = the head's 2 nf frequencies (QkRope::freqs, nf = R/4).
__global__ void __launch_bounds__(256) rope_table_kernel(const float* __restrict__ pos, const float* __restrict__ freqs,
                                                         float2* __restrict__ out, int T_tokens, int nh, int nf) {
  const int total = T_tokens * nh * 2 * nf;
  float* o = reinterpret_cast<float*>(out);
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int t = i % T_tokens;
    const int j = (i / T_tokens) % (2 * nf);
    const int h = i / (T_tokens * 2 * nf);
    float s, c;
    rope_sincos(pos[t * 2], pos[t * 2 + 1], freqs + h * 2 * nf, j, nf, s, c);
    const int64_t base = (((int64_t)h * nf + (j >> 1)) * T_tokens + t) * 4;
    o[base + (j & 1)] = c;
    o[base + 2 + (j & 1)] = s;
  }
}

int launch_rope_table(const float* pos, const float* freqs, float2* out, int T_tokens, int nh, int nf, cudaStream_t st) {
  const int total = T_tokens * nh * 2 * nf;
  rope_table_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(pos, freqs, out, T_tokens, nh, nf);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Generic attention: one warp per (batch, head, query); key set enumerated per attention type (KeySet, attn_sets.cuh).
// ------------------------------------------------------------------------------------------------

// The per-warp shared-memory slot: VECS vectors of e floats, then ARRS float arrays and one int array (the tokens) of n entries each,
// n the most keys (or queries) one warp can have.  The launcher sizes it by floats(), the kernel carves it with the accessors.
template <int VECS, int ARRS>
struct AttnSlot {
  __host__ __device__ static size_t floats(int e, int n) { return (size_t)VECS * e + (size_t)(ARRS + 1) * n; }
  float* p;
  int e, n;
  __device__ AttnSlot(float* sm, int e_, int n_) : p(sm + (threadIdx.x >> 5) * floats(e_, n_)), e(e_), n(n_) {}
  __device__ float* vec(int i) const { return p + i * e; }
  __device__ float* arr(int i) const { return p + VECS * e + i * n; }
  __device__ int* toks() const { return reinterpret_cast<int*>(arr(ARRS)); }
};

// q . k of the query qv (e floats, in shared memory) and the key row kp, fmaf in d order
template <typename T>
__device__ __forceinline__ float attn_dot(const float* qv, const T* kp, int e) {
  float s = 0.f;
  for (int d = 0; d < e; ++d) s = fmaf(qv[d], to_f(kp[d]), s);
  return s;
}

// The key walk: for the lane's keys j = lane, lane + 32, ... < nk of ks, toks[j] = the key's token (-1: masked) and sc[j] = score(j, tok)
// (-inf for a masked key, without a call).  -> the maximum score of the warp.
template <typename Score>
__device__ __forceinline__ float attn_scores(const KeySet& ks, int nk, float* sc, int* toks, Score score) {
  float mx = -INFINITY;
  for (int j0 = 0; j0 < nk; j0 += 32) {
    const int j = j0 + (threadIdx.x & 31);
    if (j < nk) {
      const int tok = ks.token(j);
      const float s = tok >= 0 ? score(j, tok) : -INFINITY;
      sc[j] = s;
      toks[j] = tok;
      mx = fmaxf(mx, s);
    }
  }
  return warp_max(mx);
}

// The softmax numerators in place of the lane's scores: p_j = exp(s_j - mx), 0 for a masked key.  -> sum_j p_j over the warp.
__device__ __forceinline__ float attn_softmax(float* sc, const int* toks, int nk, float mx) {
  float sum = 0.f;
  for (int j = threadIdx.x & 31; j < nk; j += 32) {
    const float p = (toks[j] >= 0) ? expf(sc[j] - mx) : 0.f;
    sc[j] = p;
    sum += p;
  }
  return warp_sum(sum);
}

// sum_j w_j x(j, tok_j) over the n tokens of the slot in j order, one fmaf per token, masked tokens skipped.  x reads the row of tok_j
// at the caller's dimension d; a second sum over the same tokens can ride in x.
template <typename X>
__device__ __forceinline__ float attn_wsum(const float* w, const int* toks, int n, X x) {
  float acc = 0.f;
  for (int j = 0; j < n; ++j) {
    const int tok = toks[j];
    if (tok >= 0) acc = fmaf(w[j], x(j, tok), acc);
  }
  return acc;
}

using AttnFwdSlot = AttnSlot<1, 1>;   // q | p | key tokens

template <typename T>
__global__ void __launch_bounds__(128) attn_generic_kernel(const T* __restrict__ qkv, T* __restrict__ out, int h, int w, int nh, int e,
                                                           int type, int param, int shift, int maxkeys) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31;
  const int Ttok = h * w;
  const int q = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int head = blockIdx.y;
  const int64_t b = blockIdx.z;
  const AttnFwdSlot slot(sm, e, maxkeys);
  float *qv = slot.vec(0), *sc = slot.arr(0);
  int* toks = slot.toks();
  if (q >= Ttok) return;
  const int64_t rs = 3LL * nh * e;                        // row stride of qkv
  const T* base = qkv + b * Ttok * rs;
  const T* qp = base + (int64_t)q * rs + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) qv[d] = to_f(qp[d]);
  __syncwarp();
  KeySet ks;
  ks.init(type, h, w, param, shift, q);
  const int nk = ks.count();
  const T* kb = base + (int64_t)(nh + head) * e;
  const float mx = attn_scores(ks, nk, sc, toks, [&](int, int tok) { return attn_dot(qv, kb + tok * rs, e); });
  const float inv = 1.f / attn_softmax(sc, toks, nk, mx);
  __syncwarp();
  const T* vb = base + (int64_t)(2 * nh + head) * e;
  T* op = out + (b * Ttok + q) * (int64_t)nh * e + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) op[d] = from_f<T>(attn_wsum(sc, toks, nk, [&](int, int tok) { return to_f(vb[tok * rs + d]); }) * inv);
}

// Launch of a warp-per-query (or per-key) attention kernel: a grid of (blocks of 4 warps, heads, images), the key set's geometry checked,
// and a Slot of n keys (or queries) per warp within the budget the kernel is opened to on its first launch.  Every kernel takes its
// pointers, then (h, w, nh, e, type, param, shift, n).
constexpr int kAttnSmemMax = 200 * 1024;

int check_attn_geometry(int h, int w, int type, int param) {
  if (type == KDB_ATTN_NEIGHBORHOOD) {
    KDB_REQUIRE(param >= 1 && h >= param && w >= param, KDB_ERR_BAD_SHAPE, "neighborhood attention: grid %dx%d smaller than kernel %d", h, w,
                param);
  } else if (type == KDB_ATTN_SHIFTED_WINDOW) {
    KDB_REQUIRE(param >= 1 && h % param == 0 && w % param == 0, KDB_ERR_BAD_SHAPE,
                "shifted-window attention: grid %dx%d not divisible by window %d", h, w, param);
  } else {
    KDB_REQUIRE(type == KDB_ATTN_GLOBAL, KDB_ERR_BAD_ARG, "attention: bad type %d", type);
  }
  return 0;
}

template <typename Slot>
int attn_smem(const char* what, int e, int n, size_t* smem) {
  *smem = sizeof(float) * 4 * Slot::floats(e, n);
  KDB_REQUIRE(*smem <= kAttnSmemMax, KDB_ERR_UNSUPPORTED, "%s: %d keys exceed the shared-memory budget", what, n);
  return 0;
}

template <typename Slot, auto kernel, typename... P>
int launch_attn(const char* what, int n, int B, int h, int w, int nh, int e, int type, int param, int shift, cudaStream_t st, P... ptrs) {
  static bool opened = false;
  size_t smem;
  int rc = check_attn_geometry(h, w, type, param);
  if (rc || (rc = attn_smem<Slot>(what, e, n, &smem)) || (rc = set_smem_once(kernel, opened, kAttnSmemMax))) return rc;
  kernel<<<dim3((unsigned)ceil_div(h * w, 4), (unsigned)nh, (unsigned)B), 128, smem, st>>>(ptrs..., h, w, nh, e, type, param, shift, n);
  KDB_LAUNCH_CHECK(F_ATTN_GENERIC, st);
  return 0;
}

template <typename T>
int launch_attention_generic(const T* qkv, T* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                             cudaStream_t st) {
  const int maxkeys = KeySet::count(attn_type, h, w, attn_param);
  return launch_attn<AttnFwdSlot, attn_generic_kernel<T>>("attention_generic", maxkeys, B, h, w, nh, e, attn_type, attn_param, shift, st, qkv,
                                                          out);
}
template int launch_attention_generic<float>(const float*, float*, int, int, int, int, int, int, int, int, cudaStream_t);
template int launch_attention_generic<bf16>(const bf16*, bf16*, int, int, int, int, int, int, int, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// GEGLU, TokenMerge gather
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) geglu_kernel(const T* __restrict__ h, T* __restrict__ out, int64_t M, int F) {
  const int64_t total = M * F;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t m = i / F;
    const int f = (int)(i - m * F);
    const float a = to_f(h[m * 2 * F + f]), g = to_f(h[m * 2 * F + F + f]);
    out[i] = from_f<T>(a * to_f(from_f<T>(gelu_erf(g))));
  }
}

template <typename T>
int launch_geglu(const T* h, T* out, int64_t M, int F, cudaStream_t st) {
  geglu_kernel<T><<<grid_stride_blocks(M * F), 256, 0, st>>>(h, out, M, F);
  KDB_LAUNCH_CHECK(F_GEGLU, st);
  return 0;
}
template int launch_geglu<float>(const float*, float*, int64_t, int, cudaStream_t);
template int launch_geglu<bf16>(const bf16*, bf16*, int64_t, int, cudaStream_t);

template <typename T>
__global__ void __launch_bounds__(256) merge_gather_kernel(const T* __restrict__ x, T* __restrict__ out, int H, int Wd, int C,
                                                           int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256)
    out[i] = x[merge_source(i, H / 2, Wd / 2, C)];
}

template <typename T>
int launch_merge_gather(const T* x, T* out, int B, int H, int Wd, int C, cudaStream_t st) {
  KDB_REQUIRE(H % 2 == 0 && Wd % 2 == 0, KDB_ERR_BAD_SHAPE, "token merge: grid %dx%d not even", H, Wd);
  const int64_t total = (int64_t)B * H * Wd * C;
  merge_gather_kernel<T><<<grid_stride_blocks(total), 256, 0, st>>>(x, out, H, Wd, C, total);
  KDB_LAUNCH_CHECK(F_MERGE_GATHER, st);
  return 0;
}
template int launch_merge_gather<float>(const float*, float*, int, int, int, int, cudaStream_t);
template int launch_merge_gather<bf16>(const bf16*, bf16*, int, int, int, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// out_norm + patch_out + un-patch + Karras combine.  One warp per token.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) patch_out_kernel(const T* __restrict__ tokens, const float* __restrict__ nscale,
                                                        const float* __restrict__ W, const float* __restrict__ x_in,
                                                        const float* __restrict__ sigma, float sd, float* __restrict__ out, int Cout,
                                                        int H, int Wd, int ph, int pw, int C0, int64_t tokens_total) {
  extern __shared__ float sm[];   // [warps][C0]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 4 + warp;
  if (tok >= tokens_total) return;
  float* xn = sm + (size_t)warp * C0;
  const T* xr = tokens + tok * C0;
  float ss = 0.f;
  for (int c = lane; c < C0; c += 32) {
    const float v = to_f(xr[c]);
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)C0 + kEps);
  for (int c = lane; c < C0; c += 32) xn[c] = to_f(from_f<T>(to_f(xr[c]) * (__ldg(nscale + c) * rstd)));
  __syncwarp();
  int b, ty, tx;
  token_coords(tok, H / ph, Wd / pw, b, ty, tx);
  float c_skip = 0.f, c_out = 1.f, c_in;
  if (sd > 0.f) karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
  const int N = ph * pw * Cout;
  for (int n = lane; n < N; n += 32) {
    const float* wr = W + (int64_t)n * C0;
    float acc = 0.f;
    for (int k = 0; k < C0; ++k) acc = fmaf(xn[k], __ldg(wr + k), acc);
    acc = to_f(from_f<T>(acc));
    const int64_t o = patch_pixel(b, ty, tx, n, Cout, H, Wd, ph, pw);
    out[o] = (sd > 0.f) ? acc * c_out + x_in[o] * c_skip : acc;
  }
}

template <typename T>
int launch_patch_out(const T* tokens, const float* norm_scale, const float* W, const float* x_in, const float* sigma, float sigma_data,
                     float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st) {
  {
    int rc = 0;
    if (launch_patch_out_tiled<T>(tokens, norm_scale, W, x_in, sigma, sigma_data, out, B, Cout, H, Wd, ph, pw, C0, st, &rc)) return rc;
  }
  const int64_t tok = (int64_t)B * (H / ph) * (Wd / pw);
  const size_t smem = sizeof(float) * 4 * C0;
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "patch_out: width %d too large", C0);
  patch_out_kernel<T><<<(unsigned)ceil_div(tok, 4), 128, smem, st>>>(tokens, norm_scale, W, x_in, sigma, sigma_data, out, Cout, H, Wd, ph,
                                                                     pw, C0, tok);
  KDB_LAUNCH_CHECK(F_PATCH_OUT, st);
  return 0;
}
template int launch_patch_out<float>(const float*, const float*, const float*, const float*, const float*, float, float*, int, int, int,
                                     int, int, int, int, cudaStream_t);
template int launch_patch_out<bf16>(const bf16*, const float*, const float*, const float*, const float*, float, float*, int, int, int,
                                    int, int, int, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------
// Tangent kernels of the forward-mode derivative (JVP), fp32.  Each reads the primal input of one nonlinear op and its tangent
// and writes the tangent of the op's output; the primal launch is left as it is.  Every tangent output is linear in the input
// tangent and uses only products with it, so scaling the tangent by a power of two scales the result exactly.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsnorm_jvp_kernel(const float* __restrict__ x, const float* __restrict__ dx, float* __restrict__ dy,
                                                          const float* __restrict__ scale, int64_t scale_bstride, int64_t rows_per_batch,
                                                          int64_t rows, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * C;
  const float* dr = dx + row * C;
  float ss = 0.f, sd = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = xr[c];
    ss = fmaf(v, v, ss);
    sd = fmaf(v, dr[c], sd);
  }
  const NormTangent nt(warp_sum(ss), warp_sum(sd), (float)C);
  const float* sc = scale + (row / rows_per_batch) * scale_bstride;
  float* yr = dy + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = __ldg(sc + c) * nt(xr[c], dr[c]);
}

int launch_rmsnorm_jvp(const float* x, const float* dx, float* dy, const float* scale, int64_t scale_bstride, int64_t rows_per_batch,
                       int64_t rows, int C, cudaStream_t st) {
  rmsnorm_jvp_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, st>>>(x, dx, dy, scale, scale_bstride, rows_per_batch, rows, C);
  KDB_LAUNCH_CHECK(F_RMSNORM, st);
  return 0;
}

// One warp per (token row, head) of the tangent rows; reads the un-normalised primal q, k of the same row.
__global__ void __launch_bounds__(128) qknorm_rope_jvp_kernel(const float* __restrict__ qkv, float* __restrict__ dqkv,
                                                              const float* __restrict__ pos, const QkRope qr, int64_t rows, int Ttok, int nh, int e) {
  extern __shared__ float sm[];   // [warps][2][e]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (item >= rows * nh) return;
  const int64_t row = item / nh;
  const int h = (int)(item - row * nh);
  float* buf = sm + (size_t)warp * 2 * e;
  const float py = pos[(row % Ttok) * 2 + 0], px = pos[(row % Ttok) * 2 + 1];
  const float sqs = sqrtf(qr.scale[h]);
  const float* f = qr.freqs + h * (qr.R / 2);
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int64_t off = (row * 3 + t) * (int64_t)nh * e + (int64_t)h * e;
    const float* v = qkv + off;
    float* dv = dqkv + off;
    float ss = 0.f, sd = 0.f;
    for (int d = lane; d < e; d += 32) {
      ss = fmaf(v[d], v[d], ss);
      sd = fmaf(v[d], dv[d], sd);
    }
    // the tangent of the cosine-sim scaling, then the primal's rotation
    const NormTangent nt(warp_sum(ss), warp_sum(sd), 1.f, qr.eps);
    for (int d = lane; d < e; d += 32) buf[t * e + d] = sqs * nt(v[d], dv[d]);
    __syncwarp();
    for (int d = lane; d < e; d += 32) dv[d] = rope_rotate<false>(buf + t * e, d, qr.R, py, px, f);
    __syncwarp();
  }
}

int launch_qknorm_rope_jvp(const float* qkv, float* dqkv, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e,
                           cudaStream_t st) {
  if (int rc = check_qk_rope("qknorm_rope_jvp", qr, e)) return rc;
  const size_t smem = sizeof(float) * 4 * 2 * e;
  qknorm_rope_jvp_kernel<<<(unsigned)ceil_div(rows * nh, 4), 128, smem, st>>>(qkv, dqkv, pos, qr, rows, T_tokens, nh, e);
  KDB_LAUNCH_CHECK(F_QKNORM_ROPE, st);
  return 0;
}

// Attention tangent, one warp per (batch, head, query), the key set of attn_generic_kernel:
//   do_i = sum_j P_ij dv_j + sum_j P_ij dS_ij (v_j - o_i),   dS_ij = dq_i . k_j + q_i . dk_j
using AttnJvpSlot = AttnSlot<2, 2>;   // q, dq | p, dS | key tokens

__global__ void __launch_bounds__(128) attn_jvp_kernel(const float* __restrict__ qkv, const float* __restrict__ dqkv, float* __restrict__ dout,
                                                       int h, int w, int nh, int e, int type, int param, int shift, int maxkeys) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31;
  const int Ttok = h * w;
  const int q = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int head = blockIdx.y;
  const int64_t b = blockIdx.z;
  const AttnJvpSlot slot(sm, e, maxkeys);
  float *qv = slot.vec(0), *dqv = slot.vec(1), *sc = slot.arr(0), *dsc = slot.arr(1);
  int* toks = slot.toks();
  if (q >= Ttok) return;
  const int64_t rs = 3LL * nh * e;
  const float* base = qkv + b * Ttok * rs;
  const float* dbase = dqkv + b * Ttok * rs;
  for (int d = lane; d < e; d += 32) {
    qv[d] = base[(int64_t)q * rs + (int64_t)head * e + d];
    dqv[d] = dbase[(int64_t)q * rs + (int64_t)head * e + d];
  }
  __syncwarp();
  KeySet ks;
  ks.init(type, h, w, param, shift, q);
  const int nk = ks.count();
  const float *kb = base + (int64_t)(nh + head) * e, *dkb = dbase + (int64_t)(nh + head) * e;
  const float mx = attn_scores(ks, nk, sc, toks, [&](int j, int tok) {   // s, and dS in the same loop over the key rows
    const float *kp = kb + tok * rs, *dkp = dkb + tok * rs;
    float s = 0.f, ds = 0.f;
    for (int d = 0; d < e; ++d) {
      s = fmaf(qv[d], kp[d], s);
      ds = fmaf(dqv[d], kp[d], fmaf(qv[d], dkp[d], ds));
    }
    dsc[j] = ds;
    return s;
  });
  const float inv = 1.f / attn_softmax(sc, toks, nk, mx);
  float sds = 0.f;
  for (int j = lane; j < nk; j += 32) sds = fmaf(sc[j], toks[j] >= 0 ? dsc[j] : 0.f, sds);   // dS of a masked key: never written
  const float psd = warp_sum(sds) * inv;   // sum_j P_j dS_j
  __syncwarp();
  const float *vb = base + (int64_t)(2 * nh + head) * e, *dvb = dbase + (int64_t)(2 * nh + head) * e;
  float* op = dout + (b * Ttok + q) * (int64_t)nh * e + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) {
    float o = 0.f;   // sum_j P_j v_j, in the pass of t
    const float t = attn_wsum(sc, toks, nk, [&](int j, int tok) {
      const float vv = vb[tok * rs + d];
      o = fmaf(sc[j], vv, o);
      return fmaf(dsc[j], vv, dvb[tok * rs + d]);
    });
    op[d] = t * inv - (o * inv) * psd;
  }
}

int launch_attention_jvp(const float* qkv, const float* dqkv, float* dout, int B, int h, int w, int nh, int e, int attn_type, int attn_param,
                         int shift, cudaStream_t st) {
  const int maxkeys = KeySet::count(attn_type, h, w, attn_param);
  return launch_attn<AttnJvpSlot, attn_jvp_kernel>("attention_jvp", maxkeys, B, h, w, nh, e, attn_type, attn_param, shift, st, qkv, dqkv, dout);
}

// d(a gelu(g)) = da gelu(g) + a (Phi(g) + g phi(g)) dg, erf form
__global__ void __launch_bounds__(256) geglu_jvp_kernel(const float* __restrict__ hp, const float* __restrict__ dh, float* __restrict__ dout,
                                                        int64_t M, int F) {
  const int64_t total = M * F;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t m = i / F;
    const int f = (int)(i - m * F);
    const float a = hp[m * 2 * F + f], g = hp[m * 2 * F + F + f];
    float gelu, slope;
    gelu_erf_slope(g, gelu, slope);
    dout[i] = dh[m * 2 * F + f] * gelu + (a * slope) * dh[m * 2 * F + F + f];
  }
}

int launch_geglu_jvp(const float* h, const float* dh, float* dout, int64_t M, int F, cudaStream_t st) {
  geglu_jvp_kernel<<<grid_stride_blocks(M * F), 256, 0, st>>>(h, dh, dout, M, F);
  KDB_LAUNCH_CHECK(F_GEGLU, st);
  return 0;
}

// out_norm tangent + patch_out projection + un-patch + the tangent of the Karras combine (c_skip v + c_out dF).  One warp per token.
__global__ void __launch_bounds__(128) patch_out_jvp_kernel(const float* __restrict__ tokens, const float* __restrict__ dtokens,
                                                            const float* __restrict__ nscale, const float* __restrict__ W,
                                                            const float* __restrict__ v_in, const float* __restrict__ sigma, float sd,
                                                            float* __restrict__ out, int Cout, int H, int Wd, int ph, int pw, int C0,
                                                            int64_t tokens_total) {
  extern __shared__ float sm[];   // [warps][C0]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 4 + warp;
  if (tok >= tokens_total) return;
  float* dn = sm + (size_t)warp * C0;
  const float* xr = tokens + tok * C0;
  const float* dr = dtokens + tok * C0;
  float ss = 0.f, sdot = 0.f;
  for (int c = lane; c < C0; c += 32) {
    ss = fmaf(xr[c], xr[c], ss);
    sdot = fmaf(xr[c], dr[c], sdot);
  }
  const NormTangent nt(warp_sum(ss), warp_sum(sdot), (float)C0);
  for (int c = lane; c < C0; c += 32) dn[c] = __ldg(nscale + c) * nt(xr[c], dr[c]);
  __syncwarp();
  int b, ty, tx;
  token_coords(tok, H / ph, Wd / pw, b, ty, tx);
  float c_skip = 0.f, c_out = 1.f, c_in;
  if (sd > 0.f) karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
  const int N = ph * pw * Cout;
  for (int n = lane; n < N; n += 32) {
    const float* wr = W + (int64_t)n * C0;
    float acc = 0.f;
    for (int k = 0; k < C0; ++k) acc = fmaf(dn[k], __ldg(wr + k), acc);
    const int64_t o = patch_pixel(b, ty, tx, n, Cout, H, Wd, ph, pw);
    out[o] = (sd > 0.f) ? acc * c_out + v_in[o] * c_skip : acc;
  }
}

int launch_patch_out_jvp(const float* tokens, const float* dtokens, const float* norm_scale, const float* W, const float* v_in, const float* sigma,
                         float sigma_data, float* out, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st) {
  const int64_t tok = (int64_t)B * (H / ph) * (Wd / pw);
  const size_t smem = sizeof(float) * 4 * C0;
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "patch_out_jvp: width %d too large", C0);
  patch_out_jvp_kernel<<<(unsigned)ceil_div(tok, 4), 128, smem, st>>>(tokens, dtokens, norm_scale, W, v_in, sigma, sigma_data, out, Cout, H,
                                                                      Wd, ph, pw, C0, tok);
  KDB_LAUNCH_CHECK(F_PATCH_OUT, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Backward kernels of the reverse-mode derivative (VJP), fp32.  Each reads the primal input of one op (recomputed from the tape) and
// the gradient of its output, and writes or adds the gradient of its input.  One writer per output element, no atomics, fixed
// reduction orders: two calls on the same inputs give the same bits, and every gradient is linear in the cotangent using only
// products with it, so scaling the cotangent by a power of two scales the result exactly.
// ------------------------------------------------------------------------------------------------

// dA[M,K] = dC[M,N] W[N,K] (the input gradient of C = A W^T): W is read along N, so no transposed copy exists.  The tile loop of
// simt_tile.cuh over (M, K), reducing over N.  VJP_UNPATCH_ACC: row m is a coarse token (b, hy, wx) and
// column k = (nh, nw, e); the result is added to the fine token (2hy+nh, 2wx+nw), channel e of out [B, 2hc, 2wc, Cf] -- the inverse
// of the TokenMerge gather, a bijection, so each element still has one writer.
template <int EPI>
__global__ void __launch_bounds__(256) gemm_vjp_kernel(const float* __restrict__ dC, const float* __restrict__ W, float* __restrict__ out,
                                                       int64_t M, int N, int K, int hc, int wc, int Cf) {
  const int64_t m0 = (int64_t)blockIdx.y * kTileM;
  const int k0 = blockIdx.x * kTileN;
  const int tid = threadIdx.x;
  const int lr = tid >> 2, lk = (tid & 3) * 4;    // dC loader: row 0..63, reduction offset 0,4,8,12
  const int wr = tid >> 4, wc4 = (tid & 15) * 4;  // W loader: reduction row 0..15, column offset 0..60
  auto fill = [&](int n0, TileSmem& As, TileSmem& Ws) {
    float av[4], wv[4];
    load4<float>(dC + (m0 + lr) * N + n0 + lk, (m0 + lr) < M && (n0 + lk) < N, av);
    load4<float>(W + (int64_t)(n0 + wr) * K + k0 + wc4, (n0 + wr) < N && (k0 + wc4) < K, wv);
#pragma unroll
    for (int i = 0; i < 4; ++i) As[lk + i][lr] = av[i];
    *reinterpret_cast<float4*>(&Ws[wr][wc4]) = make_float4(wv[0], wv[1], wv[2], wv[3]);
  };
  simt_tile(m0, k0, M, K, N, fill, [&](int64_t m, int k, float acc) {
    if constexpr (EPI == VJP_STORE) {
      out[m * K + k] = acc;
    } else {
      int b, hy, wx;
      token_coords(m, hc, wc, b, hy, wx);
      const int q = k / Cf, e = k - q * Cf;
      out[fine_offset(b, hy, wx, q, e, hc, wc, Cf)] += acc;
    }
  });
}

int launch_gemm_vjp(const float* dC, const float* W, float* out, int64_t M, int N, int K, int epi, int hc, int wc, int Cf, cudaStream_t st) {
  KDB_REQUIRE(N % 4 == 0 && K % 4 == 0, KDB_ERR_BAD_SHAPE, "gemm_vjp: N=%d and K=%d must be multiples of 4", N, K);
  KDB_REQUIRE(M > 0, KDB_ERR_BAD_SHAPE, "gemm_vjp: empty problem");
  KDB_REQUIRE(epi == VJP_STORE || (K == 4 * Cf && M % ((int64_t)hc * wc) == 0), KDB_ERR_BAD_SHAPE, "gemm_vjp: bad un-patch geometry");
  const int64_t chunk = 65535LL * kTileM;   // split M so gridDim.y stays legal (whole images per chunk for the un-patch epilogue)
  const int64_t step = epi == VJP_STORE ? chunk : std::max<int64_t>(chunk / ((int64_t)hc * wc), 1) * hc * wc;
  for (int64_t mo = 0; mo < M; mo += step) {
    const int64_t Mi = std::min(step, M - mo);
    dim3 grid((unsigned)ceil_div(K, kTileN), (unsigned)ceil_div(Mi, kTileM));
    KDB_REQUIRE(grid.y <= 65535u, KDB_ERR_BAD_SHAPE, "gemm_vjp: image too large");
    if (epi == VJP_STORE)
      gemm_vjp_kernel<VJP_STORE><<<grid, 256, 0, st>>>(dC + mo * N, W, out + mo * K, Mi, N, K, 0, 0, 0);
    else
      gemm_vjp_kernel<VJP_UNPATCH_ACC><<<grid, 256, 0, st>>>(dC + mo * N, W, out + mo * K, Mi, N, K, hc, wc, Cf);
    KDB_LAUNCH_CHECK(F_GEMM_SIMT, st);
  }
  return 0;
}

// dx += r (s dy) - x r^3 mean(x s dy), r = rsqrt(mean(x^2) + eps): the input gradient of (Ada)RMSNorm added to dx.  One warp per row.
__global__ void __launch_bounds__(256) rmsnorm_vjp_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                                                          const float* __restrict__ scale, int64_t scale_bstride, int64_t rows_per_batch,
                                                          int64_t rows, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * C;
  const float* gr = dy + row * C;
  const float* sc = scale + (row / rows_per_batch) * scale_bstride;
  float ss = 0.f, sd = 0.f;
  for (int c = lane; c < C; c += 32) {
    ss = fmaf(xr[c], xr[c], ss);
    sd = fmaf(xr[c], __ldg(sc + c) * gr[c], sd);
  }
  const NormTangent nt(warp_sum(ss), warp_sum(sd), (float)C);
  float* dr = dx + row * C;
  for (int c = lane; c < C; c += 32) dr[c] += nt(xr[c], __ldg(sc + c) * gr[c]);
}

int launch_rmsnorm_vjp(const float* x, const float* dy, float* dx, const float* scale, int64_t scale_bstride, int64_t rows_per_batch,
                       int64_t rows, int C, cudaStream_t st) {
  rmsnorm_vjp_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, st>>>(x, dy, dx, scale, scale_bstride, rows_per_batch, rows, C);
  KDB_LAUNCH_CHECK(F_RMSNORM, st);
  return 0;
}

// In place on the q and k thirds of dqkv: g = R(theta)^T dq^ (rotate by -theta on the primal's column pairs), then
// dq = sqrt(scale) (rho g - q rho^3 (q . g)), rho = rsqrt(sum q^2 + eps) of the un-normalised primal q in qkv.  One warp per
// (token row, head).
// dscale != nullptr: dscale[row, h] = (g_q . q rho_q + g_k . k rho_k) / (2 sqrt(scale)), the (row, head) term of d scale_h.
__global__ void __launch_bounds__(128) qknorm_rope_vjp_kernel(const float* __restrict__ qkv, float* __restrict__ dqkv,
                                                              const float* __restrict__ pos, const QkRope qr, int64_t rows, int Ttok, int nh, int e,
                                                              float* __restrict__ dscale) {
  extern __shared__ float sm[];   // [warps][e]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (item >= rows * nh) return;
  const int64_t row = item / nh;
  const int h = (int)(item - row * nh);
  float* buf = sm + (size_t)warp * e;
  const float py = pos[(row % Ttok) * 2 + 0], px = pos[(row % Ttok) * 2 + 1];
  const float sqs = sqrtf(qr.scale[h]);
  const float* f = qr.freqs + h * (qr.R / 2);
  float ds = 0.f;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int64_t off = (row * 3 + t) * (int64_t)nh * e + (int64_t)h * e;
    const float* v = qkv + off;
    float* dv = dqkv + off;
    for (int d = lane; d < e; d += 32) buf[d] = rope_rotate<true>(dv, d, qr.R, py, px, f);
    __syncwarp();
    float ss = 0.f, sg = 0.f;
    for (int d = lane; d < e; d += 32) {
      ss = fmaf(v[d], v[d], ss);
      sg = fmaf(v[d], buf[d], sg);
    }
    const float sgs = warp_sum(sg);
    const NormTangent nt(warp_sum(ss), sgs, 1.f, qr.eps);
    for (int d = lane; d < e; d += 32) dv[d] = sqs * nt(v[d], buf[d]);
    if (dscale != nullptr) ds = fmaf(sgs, nt.r, ds);
    __syncwarp();
  }
  if (dscale != nullptr && lane == 0) dscale[item] = ds / (2.f * sqs);
}

int launch_qknorm_rope_vjp(const float* qkv, float* dqkv, const float* pos, const QkRope& qr, int64_t rows, int T_tokens, int nh, int e,
                           cudaStream_t st, float* dscale_rows) {
  if (int rc = check_qk_rope("qknorm_rope_vjp", qr, e)) return rc;
  const size_t smem = sizeof(float) * 4 * e;
  qknorm_rope_vjp_kernel<<<(unsigned)ceil_div(rows * nh, 4), 128, smem, st>>>(qkv, dqkv, pos, qr, rows, T_tokens, nh, e, dscale_rows);
  KDB_LAUNCH_CHECK(F_QKNORM_ROPE, st);
  return 0;
}

// Attention VJP, query-centric pass: one warp per (batch, head, query i) over the key set of attn_generic_kernel.
//   Delta_i = dO_i . O_i,  dS_ij = P_ij (dO_i . v_j - Delta_i),  dq_i = sum_j dS_ij k_j
// It also leaves (row maximum, 1 / row sum, Delta_i) of query i in stats [B, nh, T, 3] for the key-centric pass.
using AttnVjpQSlot = AttnSlot<2, 1>;    // q, dO | p, then dS | key tokens
using AttnVjpKvSlot = AttnSlot<2, 2>;   // k, v | P, dS | query tokens

__global__ void __launch_bounds__(128) attn_vjp_q_kernel(const float* __restrict__ qkv, const float* __restrict__ o, const float* __restrict__ dout,
                                                         float* __restrict__ dqkv, float* __restrict__ stats, int h, int w, int nh, int e,
                                                         int type, int param, int shift, int maxkeys) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31;
  const int Ttok = h * w;
  const int q = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int head = blockIdx.y;
  const int64_t b = blockIdx.z;
  const AttnVjpQSlot slot(sm, e, maxkeys);
  float *qv = slot.vec(0), *dov = slot.vec(1), *sc = slot.arr(0);
  int* toks = slot.toks();
  if (q >= Ttok) return;
  const int64_t rs = 3LL * nh * e;
  const float* base = qkv + b * Ttok * rs;
  const int64_t orow = (b * Ttok + q) * (int64_t)nh * e + (int64_t)head * e;
  float delta = 0.f;
  for (int d = lane; d < e; d += 32) {
    qv[d] = base[(int64_t)q * rs + (int64_t)head * e + d];
    dov[d] = dout[orow + d];
    delta = fmaf(dov[d], o[orow + d], delta);
  }
  delta = warp_sum(delta);
  __syncwarp();
  KeySet ks;
  ks.init(type, h, w, param, shift, q);
  const int nk = ks.count();
  const float* kb = base + (int64_t)(nh + head) * e;
  const float mx = attn_scores(ks, nk, sc, toks, [&](int, int tok) { return attn_dot(qv, kb + tok * rs, e); });
  const float inv = 1.f / attn_softmax(sc, toks, nk, mx);
  for (int j = lane; j < nk; j += 32) {
    const int tok = toks[j];
    float ds = 0.f;
    if (tok >= 0) {
      const float* vp = base + (int64_t)tok * rs + (int64_t)(2 * nh + head) * e;
      float dp = 0.f;
      for (int d = 0; d < e; ++d) dp = fmaf(dov[d], vp[d], dp);
      ds = sc[j] * inv * (dp - delta);
    }
    sc[j] = ds;
  }
  __syncwarp();
  float* dq = dqkv + (b * Ttok + q) * rs + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) dq[d] = attn_wsum(sc, toks, nk, [&](int, int tok) { return kb[tok * rs + d]; });
  if (lane == 0) {
    float* st = stats + ((b * nh + head) * Ttok + q) * 3;
    st[0] = mx;
    st[1] = inv;
    st[2] = delta;
  }
}

// Attention VJP, key-centric pass: one warp per (batch, head, key j) over the queries that see key j (QuerySet).
//   dk_j = sum_i dS_ij q_i,  dv_j = sum_i P_ij dO_i
__global__ void __launch_bounds__(128) attn_vjp_kv_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ stats,
                                                          float* __restrict__ dqkv, int h, int w, int nh, int e, int type, int param, int shift,
                                                          int maxq) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31;
  const int Ttok = h * w;
  const int kt = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int head = blockIdx.y;
  const int64_t b = blockIdx.z;
  const AttnVjpKvSlot slot(sm, e, maxq);
  float *kv = slot.vec(0), *vv = slot.vec(1), *pv = slot.arr(0), *dsv = slot.arr(1);
  int* toks = slot.toks();
  if (kt >= Ttok) return;
  const int64_t rs = 3LL * nh * e;
  const float* base = qkv + b * Ttok * rs;
  for (int d = lane; d < e; d += 32) {
    kv[d] = base[(int64_t)kt * rs + (int64_t)(nh + head) * e + d];
    vv[d] = base[(int64_t)kt * rs + (int64_t)(2 * nh + head) * e + d];
  }
  __syncwarp();
  QuerySet qs;
  qs.init(type, h, w, param, shift, kt);
  const int nq = qs.count();
  const float* sb = stats + (b * nh + head) * (int64_t)Ttok * 3;
  for (int t = lane; t < nq; t += 32) {
    const int tok = qs.token(t);
    float p = 0.f, ds = 0.f;
    if (tok >= 0) {
      const float* qp = base + (int64_t)tok * rs + (int64_t)head * e;
      const float* dop = dout + (b * Ttok + tok) * (int64_t)nh * e + (int64_t)head * e;
      float s = 0.f, dp = 0.f;
      for (int d = 0; d < e; ++d) {
        s = fmaf(qp[d], kv[d], s);
        dp = fmaf(dop[d], vv[d], dp);
      }
      p = expf(s - sb[tok * 3 + 0]) * sb[tok * 3 + 1];
      ds = p * (dp - sb[tok * 3 + 2]);
    }
    pv[t] = p;
    dsv[t] = ds;
    toks[t] = tok;
  }
  __syncwarp();
  float* dk = dqkv + (b * Ttok + kt) * rs + (int64_t)(nh + head) * e;
  float* dvv = dk + (int64_t)nh * e;
  const float* qb = base + (int64_t)head * e;
  const float* dob = dout + b * Ttok * (int64_t)nh * e + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) {
    float av = 0.f;   // sum_i P_ij dO_i, in the pass of dk
    dk[d] = attn_wsum(dsv, toks, nq, [&](int t, int tok) {
      av = fmaf(pv[t], dob[tok * (int64_t)nh * e + d], av);
      return qb[tok * rs + d];
    });
    dvv[d] = av;
  }
}

int launch_attention_vjp(const float* qkv, const float* out, const float* dout, float* dqkv, float* stats, int B, int h, int w, int nh, int e,
                         int attn_type, int attn_param, int shift, cudaStream_t st) {
  const int maxkeys = KeySet::count(attn_type, h, w, attn_param), maxq = QuerySet::max_count(attn_type, h, w, attn_param);
  // the key-centric slot is the larger (maxq >= maxkeys): a shape it cannot take is refused before the first launch
  size_t smem_kv;
  int rc = check_attn_geometry(h, w, attn_type, attn_param);
  if (rc || (rc = attn_smem<AttnVjpKvSlot>("attention_vjp", e, maxq, &smem_kv)) ||
      (rc = launch_attn<AttnVjpQSlot, attn_vjp_q_kernel>("attention_vjp", maxkeys, B, h, w, nh, e, attn_type, attn_param, shift, st, qkv, out,
                                                         dout, dqkv, stats)))
    return rc;
  return launch_attn<AttnVjpKvSlot, attn_vjp_kv_kernel>("attention_vjp", maxq, B, h, w, nh, e, attn_type, attn_param, shift, st, qkv, dout,
                                                        stats, dqkv);
}

// da = dy gelu(g), dg = dy a (Phi(g) + g phi(g)), erf form; h [M, 2F] the primal up_proj output, dh [M, 2F]
__global__ void __launch_bounds__(256) geglu_vjp_kernel(const float* __restrict__ hp, const float* __restrict__ dy, float* __restrict__ dh,
                                                        int64_t M, int F) {
  const int64_t total = M * F;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t m = i / F;
    const int f = (int)(i - m * F);
    const float a = hp[m * 2 * F + f], g = hp[m * 2 * F + F + f];
    float gelu, slope;
    gelu_erf_slope(g, gelu, slope);
    dh[m * 2 * F + f] = dy[i] * gelu;
    dh[m * 2 * F + F + f] = dy[i] * (a * slope);
  }
}

int launch_geglu_vjp(const float* h, const float* dy, float* dh, int64_t M, int F, cudaStream_t st) {
  geglu_vjp_kernel<<<grid_stride_blocks(M * F), 256, 0, st>>>(h, dy, dh, M, F);
  KDB_LAUNCH_CHECK(F_GEGLU, st);
  return 0;
}

// TokenSplit VJP, elementwise part: dcur_patched = patch2x2(fac dup) -> out [B, H/2, W/2, (nh nw e)] (the TokenMerge gather order), and
// dup <- (1 - fac) dup in place (the gradient the skip connection receives).  Same derivative on both branches of lerp_torch.
__global__ void __launch_bounds__(256) split_vjp_gather_kernel(float* __restrict__ dup, float* __restrict__ out, const float* __restrict__ fac,
                                                               int H, int Wd, int C, int64_t total) {
  const float f = __ldg(fac), g = 1.f - f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t src = merge_source(i, H / 2, Wd / 2, C);
    const float d = dup[src];
    out[i] = f * d;
    dup[src] = g * d;
  }
}

int launch_split_vjp_gather(float* dup, float* out, const float* fac, int B, int H, int Wd, int C, cudaStream_t st) {
  KDB_REQUIRE(H % 2 == 0 && Wd % 2 == 0, KDB_ERR_BAD_SHAPE, "token split vjp: grid %dx%d not even", H, Wd);
  const int64_t total = (int64_t)B * H * Wd * C;
  split_vjp_gather_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(dup, out, fac, H, Wd, C, total);
  KDB_LAUNCH_CHECK(F_MERGE_GATHER, st);
  return 0;
}

// TokenSplit after a plain projection y [B, H/2, W/2, (nh nw e)]: up = lerp(skip, unpatch2x2(y), fac), as gemm_simt_kernel's
// EPI_SPLIT_LERP epilogue computes each element.  One thread per element, coarse index i in the TokenMerge order.
__global__ void __launch_bounds__(256) split_unpatch_lerp_kernel(const float* __restrict__ y, const float* __restrict__ skip,
                                                                 const float* __restrict__ fac, float* __restrict__ up, int H, int Wd, int C,
                                                                 int64_t total) {
  const float f = __ldg(fac);
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t dst = merge_source(i, H / 2, Wd / 2, C);
    up[dst] = lerp_torch(skip[dst], y[i], f);
  }
}

int launch_split_unpatch_lerp(const float* y, const float* skip, const float* fac, float* up, int B, int H, int Wd, int C, cudaStream_t st) {
  KDB_REQUIRE(H % 2 == 0 && Wd % 2 == 0, KDB_ERR_BAD_SHAPE, "token split: grid %dx%d not even", H, Wd);
  const int64_t total = (int64_t)B * H * Wd * C;
  split_unpatch_lerp_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(y, skip, fac, up, H, Wd, C, total);
  KDB_LAUNCH_CHECK(F_MERGE_GATHER, st);
  return 0;
}

// TokenMerge VJP after a plain input-gradient GEMM d [B, H/2, W/2, (nh nw e)]: dfine += unpatch2x2(d).  The map is a bijection, so each
// fine element is read and written by one thread.
__global__ void __launch_bounds__(256) merge_scatter_add_kernel(const float* __restrict__ d, float* __restrict__ dfine, int H, int Wd, int C,
                                                                int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t dst = merge_source(i, H / 2, Wd / 2, C);
    dfine[dst] += d[i];
  }
}

int launch_merge_scatter_add(const float* d, float* dfine, int B, int H, int Wd, int C, cudaStream_t st) {
  KDB_REQUIRE(H % 2 == 0 && Wd % 2 == 0, KDB_ERR_BAD_SHAPE, "token merge vjp: grid %dx%d not even", H, Wd);
  const int64_t total = (int64_t)B * H * Wd * C;
  merge_scatter_add_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(d, dfine, H, Wd, C, total);
  KDB_LAUNCH_CHECK(F_MERGE_GATHER, st);
  return 0;
}

// patch_out + out_norm VJP: per token, dy = patch(c_out u) (c_out = 1 for the raw model), dxn = dy W_po, dt = RMSNorm_vjp(tokens, dxn)
// written to dtokens.  One warp per token.
__global__ void __launch_bounds__(128) patch_out_vjp_kernel(const float* __restrict__ tokens, const float* __restrict__ nscale,
                                                            const float* __restrict__ W, const float* __restrict__ u, const float* __restrict__ sigma,
                                                            float sd, float* __restrict__ dtokens, int Cout, int H, int Wd, int ph, int pw,
                                                            int C0, int64_t tokens_total, float* __restrict__ dnorm, float* __restrict__ rstd) {
  extern __shared__ float sm[];   // [warps][C0 + N]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tok = (int64_t)blockIdx.x * 4 + warp;
  if (tok >= tokens_total) return;
  const int N = ph * pw * Cout;
  float* dn = sm + (size_t)warp * (C0 + N);
  float* dy = dn + C0;
  int b, ty, tx;
  token_coords(tok, H / ph, Wd / pw, b, ty, tx);
  float c_skip, c_out = 1.f, c_in;
  if (sd > 0.f) karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
  for (int n = lane; n < N; n += 32) dy[n] = c_out * u[patch_pixel(b, ty, tx, n, Cout, H, Wd, ph, pw)];
  __syncwarp();
  for (int k = lane; k < C0; k += 32) {
    float acc = 0.f;
    for (int n = 0; n < N; ++n) acc = fmaf(dy[n], __ldg(W + (int64_t)n * C0 + k), acc);
    dn[k] = acc;
  }
  __syncwarp();
  const float* xr = tokens + tok * C0;
  float ss = 0.f, sdot = 0.f;
  for (int c = lane; c < C0; c += 32) {
    ss = fmaf(xr[c], xr[c], ss);
    sdot = fmaf(xr[c], __ldg(nscale + c) * dn[c], sdot);
  }
  const NormTangent nt(warp_sum(ss), warp_sum(sdot), (float)C0);
  float* dr = dtokens + tok * C0;
  for (int c = lane; c < C0; c += 32) dr[c] = nt(xr[c], __ldg(nscale + c) * dn[c]);
  if (dnorm != nullptr)
    for (int c = lane; c < C0; c += 32) dnorm[tok * C0 + c] = dn[c];
  if (rstd != nullptr && lane == 0) rstd[tok] = nt.r;
}

int launch_patch_out_vjp(const float* tokens, const float* norm_scale, const float* W, const float* u, const float* sigma, float sigma_data,
                         float* dtokens, int B, int Cout, int H, int Wd, int ph, int pw, int C0, cudaStream_t st, float* dnorm, float* rstd) {
  const int64_t tok = (int64_t)B * (H / ph) * (Wd / pw);
  const size_t smem = sizeof(float) * 4 * (size_t)(C0 + ph * pw * Cout);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "patch_out_vjp: width %d too large", C0);
  patch_out_vjp_kernel<<<(unsigned)ceil_div(tok, 4), 128, smem, st>>>(tokens, norm_scale, W, u, sigma, sigma_data, dtokens, Cout, H, Wd, ph, pw,
                                                                      C0, tok, dnorm, rstd);
  KDB_LAUNCH_CHECK(F_PATCH_OUT, st);
  return 0;
}

// patch_in VJP with the Karras combine's skip term: grad_x = c_skip u + c_in unpatch(dt0 W_pi) (sigma_data > 0), else unpatch(dt0 W_pi).
// One thread per input element; W_pi [N, K] with K = (nh, nw, c).
__global__ void __launch_bounds__(256) patch_in_vjp_kernel(const float* __restrict__ dtok, const float* __restrict__ W, const float* __restrict__ u,
                                                           const float* __restrict__ sigma, float sd, float* __restrict__ grad, int C, int H, int Wd,
                                                           int ph, int pw, int N, int64_t total) {
  const int K = ph * pw * C;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int xx = (int)(i % Wd);
    int64_t r = i / Wd;
    const int y = (int)(r % H);
    r /= H;
    const int c = (int)(r % C);
    const int64_t b = r / C;
    const int64_t tok = (b * (H / ph) + y / ph) * (Wd / pw) + xx / pw;
    const int k = ((y % ph) * pw + (xx % pw)) * C + c;
    const float* dr = dtok + tok * N;
    float acc = 0.f;
    for (int n = 0; n < N; ++n) acc = fmaf(dr[n], __ldg(W + (int64_t)n * K + k), acc);
    if (sd > 0.f) {
      float c_skip, c_out, c_in;
      karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
      acc = c_skip * u[i] + c_in * acc;
    }
    grad[i] = acc;
  }
}

int launch_patch_in_vjp(const float* dtokens, const float* W, const float* u, const float* sigma, float sigma_data, float* grad_x, int B, int C,
                        int H, int Wd, int ph, int pw, int N, cudaStream_t st) {
  const int64_t total = (int64_t)B * C * H * Wd;
  patch_in_vjp_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(dtokens, W, u, sigma, sigma_data, grad_x, C, H, Wd, ph, pw, N, total);
  KDB_LAUNCH_CHECK(F_PATCH_IN, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Conditioning: FourierFeatures -> in-proj -> MappingNetwork -> concatenated AdaRMSNorm projections.
// One CTA (8 warps) per row; warp-per-output matvecs, weights streamed from L2.
// ------------------------------------------------------------------------------------------------
// vout[o] = (accumulate ? vout[o] : 0) + bias + W[o, :] . vin for o in [o_begin, o_end).  One warp per output, four outputs
// in flight per warp and 16-byte weight loads, so a warp keeps 8+ independent L2 requests outstanding (the chain of
// matvecs is latency bound, not bandwidth bound).
__device__ __forceinline__ void block_matvec(const float* __restrict__ W, const float* vin, float* vout, int o_begin, int o_end, int n_in,
                                             bool accumulate, float bias = 0.f) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const bool vec = (n_in % 128 == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  for (int o = o_begin + warp; o < o_end; o += 4 * nw) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    if (vec) {
      for (int k = lane * 4; k < n_in; k += 128) {
        const float4 x = *reinterpret_cast<const float4*>(vin + k);
        float4 wv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int oo = o + u * nw;
          wv[u] = oo < o_end ? __ldg(reinterpret_cast<const float4*>(W + (int64_t)oo * n_in + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) s[u] = fmaf(wv[u].x, x.x, fmaf(wv[u].y, x.y, fmaf(wv[u].z, x.z, fmaf(wv[u].w, x.w, s[u]))));
      }
    } else {
      for (int k = lane; k < n_in; k += 32) {
        const float x = vin[k];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int oo = o + u * nw;
          if (oo < o_end) s[u] = fmaf(__ldg(W + (int64_t)oo * n_in + k), x, s[u]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int oo = o + u * nw;
      const float t = warp_sum(s[u]);
      if (lane == 0 && oo < o_end) vout[oo] = (accumulate ? vout[oo] : 0.f) + bias + t;
    }
  }
}

// y = x * scale * rsqrt(mean(x^2) + eps), vectors in shared memory
__device__ __forceinline__ void block_rmsnorm(const float* x, float* y, const float* __restrict__ scale, int n, float* red) {
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) ss = fmaf(x[i], x[i], ss);
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)n + kEps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = x[i] * (__ldg(scale + i) * rstd);
  __syncthreads();
}

// Where map_forward leaves each activation of one conditioning row.  The conditioning kernel aliases them onto a few shared-memory
// vectors (every r[l] is one in-place stream, g[l] overwrites up[l]); the mapping backward gives each its own slot of a MapLayout row.
struct MapBufs {
  float *ff_t, *ff_a, *emb, *mc, *red, *cond;
  float *r[9], *xn[8], *up[8], *g[8];
};

// FourierFeatures -> in-proj -> MappingNetwork of conditioning row `row` (image_transformer_v2.py:552-581,734-740): cond = b.cond
__device__ void map_forward(const CondWeights& w, int row, const float* __restrict__ sigma, const float* __restrict__ aug,
                            const int64_t* __restrict__ cls, const float* __restrict__ mcond, const MapBufs& b) {
  const int mw = w.mw, dff = w.dff;
  const int half = mw / 2;
  const float two_pi = 6.283185307179586f;

  // time embedding: FourierFeatures(log(sigma)/4) -> time_in_proj        (:734-735, layers.py:291-293)
  const float c_noise = logf(sigma[row]) / 4.f;
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    const float f = (two_pi * c_noise) * __ldg(w.time_emb + j);
    float s, c;
    sincosf(f, &s, &c);
    b.ff_t[j] = c;
    b.ff_t[half + j] = s;
  }
  __syncthreads();
  block_matvec(w.time_in, b.ff_t, b.emb, 0, mw, mw, false);
  __syncthreads();
  // augmentation embedding (zeros when aug_cond is None, :736-737)
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    float f = 0.f;
    if (aug != nullptr)
      for (int k = 0; k < 9; ++k) f = fmaf(two_pi * aug[(int64_t)row * 9 + k], __ldg(w.aug_emb + j * 9 + k), f);
    float s, c;
    sincosf(f, &s, &c);
    b.ff_a[j] = c;
    b.ff_a[half + j] = s;
  }
  __syncthreads();
  block_matvec(w.aug_in, b.ff_a, b.emb, 0, mw, mw, true);
  __syncthreads();
  if (w.class_emb != nullptr) {
    const int64_t ci = cls[row];
    for (int j = threadIdx.x; j < mw; j += blockDim.x) b.emb[j] += __ldg(w.class_emb + ci * mw + j);
  }
  if (w.mcond_in != nullptr) {
    for (int j = threadIdx.x; j < w.mcond_dim; j += blockDim.x) b.mc[j] = mcond[(int64_t)row * w.mcond_dim + j];
    __syncthreads();
    block_matvec(w.mcond_in, b.mc, b.emb, 0, mw, w.mcond_dim, true);
  }
  __syncthreads();

  // MappingNetwork (:569-581)
  block_rmsnorm(b.emb, b.r[0], w.in_norm, mw, b.red);
  for (int l = 0; l < w.depth; ++l) {
    block_rmsnorm(b.r[l], b.xn[l], w.blk_norm[l], mw, b.red);
    block_matvec(w.blk_up[l], b.xn[l], b.up[l], 0, 2 * dff, mw, false);
    __syncthreads();
    for (int i = threadIdx.x; i < dff; i += blockDim.x) b.g[l][i] = b.up[l][i] * gelu_erf(b.up[l][dff + i]);
    if (b.r[l + 1] != b.r[l])
      for (int i = threadIdx.x; i < mw; i += blockDim.x) b.r[l + 1][i] = b.r[l][i];
    __syncthreads();
    block_matvec(w.blk_down[l], b.g[l], b.r[l + 1], 0, mw, dff, true);
    __syncthreads();
  }
  block_rmsnorm(b.r[w.depth], b.cond, w.out_norm, mw, b.red);
}

__global__ void __launch_bounds__(256) conditioning_kernel(const CondWeights w, const float* __restrict__ sigma,
                                                           const float* __restrict__ aug, const int64_t* __restrict__ cls,
                                                           const float* __restrict__ mcond, float* __restrict__ out, int64_t out_stride) {
  extern __shared__ float4 cond_sm4[];          // 16-byte aligned: block_matvec reads its input vector as float4
  float* sm = reinterpret_cast<float*>(cond_sm4);
  const int mw = w.mw, dff = w.dff;
  MapBufs b;
  b.ff_t = b.ff_a = sm;        // [mw]   fourier features
  b.emb = b.ff_t + mw;         // [mw]   summed embedding / residual stream
  float* xn = b.emb + mw;      // [mw]
  float* up = xn + mw;         // [2*dff]
  b.red = up + 2 * dff;        // [32]
  b.mc = b.red + 32;           // [mcond_dim]
  b.cond = xn;
  for (int l = 0; l <= 8; ++l) b.r[l] = b.emb;
  for (int l = 0; l < 8; ++l) {
    b.xn[l] = xn;
    b.up[l] = b.g[l] = up;
  }
  const int row = blockIdx.x;
  map_forward(w, row, sigma, aug, cls, mcond, b);

  // every AdaRMSNorm: scale = Linear(cond) + 1   (:166).  The CTAs of one row (gridDim.y) share the outputs; each repeats the
  // (short) mapping network so that no second launch or grid-wide hand-off is needed.
  float* orow = out + (int64_t)row * out_stride;
  const int per = (w.ada_total + (int)gridDim.y - 1) / (int)gridDim.y;
  const int o0 = (int)blockIdx.y * per, o1 = min(w.ada_total, o0 + per);
  block_matvec(w.ada_cat, xn, orow, o0, o1, mw, false, 1.f);
  if (blockIdx.y == 0)
    for (int j = threadIdx.x; j < mw; j += blockDim.x) orow[w.ada_total + j] = xn[j];   // cond itself (debug / taps)
}

int launch_conditioning(const CondWeights& w, int rows, const float* sigma, const float* aug, const int64_t* cls, const float* mcond,
                        float* out, int64_t out_stride, cudaStream_t st) {
  KDB_REQUIRE(w.mw % 4 == 0 && w.dff % 2 == 0 && w.depth <= 8, KDB_ERR_UNSUPPORTED, "conditioning: mapping width must be a multiple of 4, depth <= 8");
  const size_t smem = sizeof(float) * (size_t)(3 * w.mw + 2 * w.dff + 32 + w.mcond_dim);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "conditioning: mapping network too wide");
  conditioning_kernel<<<dim3((unsigned)rows, 4), 256, smem, st>>>(w, sigma, aug, cls, mcond, out, out_stride);
  KDB_LAUNCH_CHECK(F_COND, st);
  return 0;
}

// dx (+)= the input gradient of y = x * scale * rsqrt(mean(x^2) + eps) (block_rmsnorm) for the output gradient dy, vectors of n
__device__ __forceinline__ void block_rmsnorm_vjp(const float* x, const float* dy, const float* __restrict__ scale, float* dx, int n, float* red,
                                                  bool accumulate) {
  float ss = 0.f, sd = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    ss = fmaf(x[i], x[i], ss);
    sd = fmaf(x[i], __ldg(scale + i) * dy[i], sd);
  }
  ss = block_sum(ss, red);
  sd = block_sum(sd, red);
  const NormTangent nt(ss, sd, (float)n);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = nt(x[i], __ldg(scale + i) * dy[i]);
    dx[i] = accumulate ? dx[i] + v : v;
  }
  __syncthreads();
}

// vout[k] = sum over o < n_rows of W[o, k] vin[o] for k < n_cols (the input gradient of block_matvec), o in order
__device__ __forceinline__ void block_matvec_t(const float* __restrict__ W, const float* vin, float* vout, int n_rows, int n_cols) {
  for (int k = threadIdx.x; k < n_cols; k += blockDim.x) {
    float s = 0.f;
    for (int o = 0; o < n_rows; ++o) s = fmaf(__ldg(W + (int64_t)o * n_cols + k), vin[o], s);
    vout[k] = s;
  }
}

// One CTA per conditioning row: map_forward into the row's MapLayout slots of keep, then the reverse walk out_norm, the blocks (last
// first), in_norm, from dcond into the row of grad.
__global__ void __launch_bounds__(256) mapping_backward_kernel(const CondWeights w, const MapLayout L, const float* __restrict__ sigma,
                                                               const float* __restrict__ aug, const int64_t* __restrict__ cls,
                                                               const float* __restrict__ mcond, const float* __restrict__ dcond,
                                                               float* __restrict__ keep, float* __restrict__ grad) {
  extern __shared__ float4 map_bwd_sm4[];
  float* sm = reinterpret_cast<float*>(map_bwd_sm4);
  const int mw = w.mw, dff = w.dff, D = w.depth;
  const int row = blockIdx.x;
  float* k = keep + (int64_t)row * L.keep_floats();
  float* g = grad + (int64_t)row * L.grad_floats();
  MapBufs b;
  b.mc = sm;                                     // [mcond_dim], 16-byte aligned for block_matvec
  b.red = sm + ((w.mcond_dim + 3) & ~3);         // [32]
  float* dg = b.red + 32;                        // [dff]
  b.ff_t = k + L.ff_t();
  b.ff_a = k + L.ff_a();
  b.emb = k + L.emb();
  b.cond = g + L.demb();                         // the recomputed cond is not needed: scratch until demb is written
  for (int l = 0; l <= D; ++l) b.r[l] = k + L.r(l);
  for (int l = 0; l < D; ++l) {
    b.xn[l] = k + L.xn(l);
    b.up[l] = k + L.up(l);
    b.g[l] = k + L.g(l);
  }
  map_forward(w, row, sigma, aug, cls, mcond, b);

  block_rmsnorm_vjp(b.r[D], dcond + (int64_t)row * mw, w.out_norm, g + L.dr(D), mw, b.red, false);
  for (int l = D - 1; l >= 0; --l) {
    const float* dr1 = g + L.dr(l + 1);
    float *dxn = g + L.dxn(l), *dh = g + L.dh(l), *dr = g + L.dr(l);
    block_matvec_t(w.blk_down[l], dr1, dg, mw, dff);
    __syncthreads();
    for (int i = threadIdx.x; i < dff; i += blockDim.x) {   // GEGLU backward, as geglu_vjp_kernel
      float gelu, slope;
      gelu_erf_slope(b.up[l][dff + i], gelu, slope);
      dh[i] = dg[i] * gelu;
      dh[dff + i] = dg[i] * (b.up[l][i] * slope);
    }
    for (int i = threadIdx.x; i < mw; i += blockDim.x) dr[i] = dr1[i];   // the residual branch
    __syncthreads();
    block_matvec_t(w.blk_up[l], dh, dxn, 2 * dff, mw);
    __syncthreads();
    block_rmsnorm_vjp(b.r[l], dxn, w.blk_norm[l], dr, mw, b.red, true);
  }
  block_rmsnorm_vjp(b.emb, g + L.dr(0), w.in_norm, g + L.demb(), mw, b.red, false);
}

int launch_mapping_backward(const CondWeights& w, int rows, const float* sigma, const float* aug, const int64_t* cls, const float* mcond,
                            const float* dcond, float* keep, float* grad, cudaStream_t st) {
  KDB_REQUIRE(w.mw % 4 == 0 && w.dff % 2 == 0 && w.depth <= 8, KDB_ERR_UNSUPPORTED, "mapping backward: mapping width must be a multiple of 4, depth <= 8");
  const size_t smem = sizeof(float) * (size_t)(((w.mcond_dim + 3) & ~3) + 32 + w.dff);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "mapping backward: mapping network too wide");
  mapping_backward_kernel<<<(unsigned)rows, 256, smem, st>>>(w, MapLayout{w.mw, w.dff, w.depth}, sigma, aug, cls, mcond, dcond, keep, grad);
  KDB_LAUNCH_CHECK(F_COND, st);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// dtype conversion
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) out[i] = __float2bfloat16_rn(in[i]);
}
int launch_f32_to_bf16(const float* in, bf16* out, int64_t n, cudaStream_t st) {
  f32_to_bf16_kernel<<<grid_stride_blocks(n), 256, 0, st>>>(in, out, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

template <typename T>
__global__ void __launch_bounds__(256) to_f32_kernel(const T* __restrict__ in, float* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) out[i] = to_f(in[i]);
}
template <typename T>
int launch_to_f32(const T* in, float* out, int64_t n, cudaStream_t st) {
  to_f32_kernel<T><<<grid_stride_blocks(n), 256, 0, st>>>(in, out, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}
template int launch_to_f32<float>(const float*, float*, int64_t, cudaStream_t);
template int launch_to_f32<bf16>(const bf16*, float*, int64_t, cudaStream_t);

}  // namespace kdb
