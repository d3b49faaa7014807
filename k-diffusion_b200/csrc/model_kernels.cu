// model_kernels.cu -- precision-templated SIMT kernels for every op of the image_transformer_v2
// forward pass (reference: k_diffusion/models/image_transformer_v2.py).  With T = float this is the
// fp32-exact path behind the rtol 1e-3 / atol 1e-5 parity gate: all reductions accumulate in fp32,
// transcendental functions are the accurate (non fast-math) variants.  With T = bf16 the same
// kernels serve as the fallback for shapes the tensor-core (wgmma) kernels do not cover.
#include <cmath>

#include "model_kernels.cuh"

namespace kdb {

constexpr float kEps = 1e-6f;   // RMSNorm / cosine-sim eps (image_transformer_v2.py:143,378)

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
      const int b = (int)(tok / ((int64_t)th_n * tw_n));
      const int r = (int)(tok - (int64_t)b * th_n * tw_n);
      const int ty = r / tw_n, tx = r - ty * tw_n;
      const int nh = k / (pw * C), nw = (k / C) % pw, c = k % C;
      float c_in = 1.f;
      if (sd > 0.f) {
        float cs, co;
        karras_scalings(sigma[b], sd, cs, co, c_in);
      }
      v = x[(((int64_t)b * C + c) * H + (ty * ph + nh)) * Wd + (tx * pw + nw)] * c_in;
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
// SIMT GEMM, C = A W^T, fp32 accumulate.  64x64x16 tiles, 256 threads, 4x4 micro-tile per thread.
// ------------------------------------------------------------------------------------------------
constexpr int GBM = 64, GBN = 64, GBK = 16, GPAD = 4;

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

__device__ __forceinline__ float lerp_like_torch(float start, float end, float w) {
  // ATen lerp: w < 0.5 ? start + w (end - start) : end - (end - start)(1 - w)
  const float d = end - start;
  return (w < 0.5f) ? fmaf(w, d, start) : end - d * (1.f - w);
}

template <typename T, typename TW, int EPI>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const T* __restrict__ A, const TW* __restrict__ W, T* __restrict__ Cout,
                                                        int64_t M, int N, int K, const T* __restrict__ resid,
                                                        const float* __restrict__ fac, int hc, int wc, int Cf) {
  __shared__ __align__(16) float As[GBK][GBM + GPAD];
  __shared__ __align__(16) float Ws[GBK][GBN + GPAD];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.y * GBM;
  const int n0 = blockIdx.x * GBN;
  const int lr = tid >> 2, lk = (tid & 3) * 4;   // loader: row 0..63, k offset 0,4,8,12
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += GBK) {
    float av[4], wv[4];
    load4<T>(A + (m0 + lr) * K + k0 + lk, (m0 + lr) < M && (k0 + lk) < K, av);
    load4<TW>(W + (int64_t)(n0 + lr) * K + k0 + lk, (n0 + lr) < N && (k0 + lk) < K, wv);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[lk + i][lr] = av[i];
      Ws[lk + i][lr] = wv[i];
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GBK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Ws[kk][tx * 4]);
      const float aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }

  float facv = 0.f;
  if constexpr (EPI == EPI_SPLIT_LERP) facv = __ldg(fac);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      if constexpr (EPI == EPI_STORE) {
        Cout[m * N + n] = from_f<T>(acc[i][j]);
      } else if constexpr (EPI == EPI_RESID) {
        Cout[m * N + n] = from_f<T>(acc[i][j] + to_f(resid[m * N + n]));
      } else {
        // TokenSplit: row m = (b, hy, wx) on the coarse grid, column n = (nh, nw, e)
        const int64_t b = m / ((int64_t)hc * wc);
        const int r = (int)(m - b * hc * wc);
        const int hy = r / wc, wx = r - hy * wc;
        const int q = n / Cf, e = n - q * Cf;
        const int nh = q >> 1, nw = q & 1;
        const int64_t dst = ((b * (2 * hc) + (2 * hy + nh)) * (2 * wc) + (2 * wx + nw)) * Cf + e;
        Cout[dst] = from_f<T>(lerp_like_torch(to_f(resid[dst]), acc[i][j], facv));
      }
    }
  }
}

template <typename T, typename TW>
int launch_gemm_simt(const T* A, const TW* W, T* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st) {
  KDB_REQUIRE(K % 4 == 0, KDB_ERR_BAD_SHAPE, "gemm_simt: K=%d must be a multiple of 4", K);
  KDB_REQUIRE(M > 0 && N > 0, KDB_ERR_BAD_SHAPE, "gemm_simt: empty problem");
  dim3 grid((unsigned)ceil_div(N, GBN), (unsigned)ceil_div(M, GBM));
  KDB_REQUIRE(grid.y <= 65535u * 16u, KDB_ERR_BAD_SHAPE, "gemm_simt: M too large");
  if (grid.y > 65535u) {   // split M so gridDim.y stays legal
    const int64_t chunk = 65535LL * GBM;
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
// cosine-sim scaling + axial RoPE, in place on q and k.  One warp per (token row, head).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) qknorm_rope_kernel(T* __restrict__ qkv, const float* __restrict__ pos,
                                                          const float* __restrict__ freqs, const float* __restrict__ scale,
                                                          int64_t rows, int Ttok, int nh, int e) {
  extern __shared__ float sm[];   // [warps][2][e]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (item >= rows * nh) return;
  const int64_t row = item / nh;
  const int h = (int)(item - row * nh);
  float* buf = sm + (size_t)warp * 2 * e;
  const int dr = e / 4;        // rotated pair width: theta has 2 * (e/8) entries (AxialRoPE(d_head // 2))
  const int nf = e / 8;
  const float py = pos[(row % Ttok) * 2 + 0], px = pos[(row % Ttok) * 2 + 1];
  const float sqs = sqrtf(scale[h]);
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    T* v = qkv + (row * 3 + t) * (int64_t)nh * e + (int64_t)h * e;
    float ss = 0.f;
    for (int d = lane; d < e; d += 32) {
      const float f = to_f(v[d]);
      ss = fmaf(f, f, ss);
    }
    ss = warp_sum(ss);
    const float sc = sqs * rsqrtf(ss + kEps);
    // the reference rounds the scaled q/k back to the activation dtype before RoPE (:114)
    for (int d = lane; d < e; d += 32) buf[t * e + d] = to_f(from_f<T>(to_f(v[d]) * sc));
    __syncwarp();
    for (int d = lane; d < e; d += 32) {
      float o;
      if (d < 2 * dr) {
        const int j = d < dr ? d : d - dr;
        const float theta = (j < nf ? py : px) * freqs[h * nf + (j < nf ? j : j - nf)];
        float s, c;
        sincosf(theta, &s, &c);
        const float x1 = buf[t * e + j], x2 = buf[t * e + j + dr];
        o = d < dr ? x1 * c - x2 * s : x2 * c + x1 * s;
      } else {
        o = buf[t * e + d];
      }
      v[d] = from_f<T>(o);
    }
    __syncwarp();
  }
}

template <typename T>
int launch_qknorm_rope(T* qkv, const float* pos, const float* freqs, const float* scale, int64_t rows, int T_tokens, int nh, int e,
                       cudaStream_t st) {
  KDB_REQUIRE(e % 8 == 0, KDB_ERR_BAD_SHAPE, "qknorm_rope: d_head %d must be a multiple of 8", e);
  const size_t smem = sizeof(float) * 4 * 2 * e;
  qknorm_rope_kernel<T><<<(unsigned)ceil_div(rows * nh, 4), 128, smem, st>>>(qkv, pos, freqs, scale, rows, T_tokens, nh, e);
  KDB_LAUNCH_CHECK(F_QKNORM_ROPE, st);
  return 0;
}
template int launch_qknorm_rope<float>(float*, const float*, const float*, const float*, int64_t, int, int, int, cudaStream_t);
template int launch_qknorm_rope<bf16>(bf16*, const float*, const float*, const float*, int64_t, int, int, int, cudaStream_t);

// RoPE table for the QKV epilogue: float4 [(head * nf + i) * T + token] = (cos t_2i, cos t_2i+1, sin t_2i, sin t_2i+1), i < nf.
// Token-minor, so the 32 threads of an epilogue warp (32 consecutive tokens) read 512 contiguous bytes per load, and the
// (cos, cos, sin, sin) order is what the packed-fp32 rotation consumes.  theta_j = pos_h * f_j (j < nf) or pos_w * f_{j-nf}.
__global__ void __launch_bounds__(256) rope_table_kernel(const float* __restrict__ pos, const float* __restrict__ freqs,
                                                         float2* __restrict__ out, int T_tokens, int nh, int nf) {
  const int total = T_tokens * nh * 2 * nf;
  float* o = reinterpret_cast<float*>(out);
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int t = i % T_tokens;
    const int j = (i / T_tokens) % (2 * nf);
    const int h = i / (T_tokens * 2 * nf);
    const float theta = (j < nf ? pos[t * 2] : pos[t * 2 + 1]) * freqs[h * nf + (j < nf ? j : j - nf)];
    float s, c;
    sincosf(theta, &s, &c);
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
// Generic attention: one warp per (batch, head, query); key set enumerated per attention type.
// ------------------------------------------------------------------------------------------------
struct KeySet {
  int type, h, w, param, shift;
  int qi, qj;           // query coordinates
  int r0, c0;           // neighbourhood origin
  int wi, wj, lqi, lqj; // shifted-window: window index and local query coords (rolled frame)
  __device__ int count() const { return type == KDB_ATTN_GLOBAL ? h * w : param * param; }
  __device__ void init(int type_, int h_, int w_, int param_, int shift_, int q) {
    type = type_; h = h_; w = w_; param = param_; shift = shift_;
    qi = q / w; qj = q - qi * w;
    if (type == KDB_ATTN_NEIGHBORHOOD) {
      r0 = min(max(qi - param / 2, 0), h - param);
      c0 = min(max(qj - param / 2, 0), w - param);
    } else if (type == KDB_ATTN_SHIFTED_WINDOW) {
      const int ri = (qi + shift) % h, rj = (qj + shift) % w;   // position in the rolled image (:274)
      wi = ri / param; wj = rj / param; lqi = ri - wi * param; lqj = rj - wj * param;
    }
  }
  // token index of key j, or -1 if masked out
  __device__ int token(int j) const {
    if (type == KDB_ATTN_GLOBAL) return j;
    const int a = j / param, b = j - a * param;
    if (type == KDB_ATTN_NEIGHBORHOOD) return (r0 + a) * w + (c0 + b);
    if (shift > 0) {   // seam mask (:300-315): only the first window row/col contains wrapped tokens
      if (wi == 0 && ((lqi < shift) != (a < shift))) return -1;
      if (wj == 0 && ((lqj < shift) != (b < shift))) return -1;
    }
    const int oi = (wi * param + a - shift + h) % h, oj = (wj * param + b - shift + w) % w;
    return oi * w + oj;
  }
};

template <typename T>
__global__ void __launch_bounds__(128) attn_generic_kernel(const T* __restrict__ qkv, T* __restrict__ out, int h, int w, int nh, int e,
                                                           int type, int param, int shift, int maxkeys) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Ttok = h * w;
  const int q = blockIdx.x * 4 + warp;
  const int head = blockIdx.y;
  const int64_t b = blockIdx.z;
  float* qv = sm + (size_t)warp * (e + 2 * maxkeys);
  float* sc = qv + e;
  int* toks = reinterpret_cast<int*>(sc + maxkeys);
  if (q >= Ttok) return;
  const int64_t rs = 3LL * nh * e;                        // row stride of qkv
  const T* base = qkv + b * Ttok * rs;
  const T* qp = base + (int64_t)q * rs + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) qv[d] = to_f(qp[d]);
  __syncwarp();
  KeySet ks;
  ks.init(type, h, w, param, shift, q);
  const int nk = ks.count();
  float mx = -INFINITY;
  for (int j0 = 0; j0 < nk; j0 += 32) {
    const int j = j0 + lane;
    if (j < nk) {
      const int tok = ks.token(j);
      float s = -INFINITY;
      if (tok >= 0) {
        const T* kp = base + (int64_t)tok * rs + (int64_t)(nh + head) * e;
        s = 0.f;
        for (int d = 0; d < e; ++d) s = fmaf(qv[d], to_f(kp[d]), s);
      }
      sc[j] = s;
      toks[j] = tok;
      mx = fmaxf(mx, s);
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
  __syncwarp();
  for (int j = lane; j < nk; j += 32) {
    const float p = (toks[j] >= 0) ? expf(sc[j] - mx) : 0.f;
    sc[j] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.f / sum;
  T* op = out + (b * Ttok + q) * (int64_t)nh * e + (int64_t)head * e;
  for (int d = lane; d < e; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < nk; ++j) {
      const int tok = toks[j];
      if (tok >= 0) acc = fmaf(sc[j], to_f(base[(int64_t)tok * rs + (int64_t)(2 * nh + head) * e + d]), acc);
    }
    op[d] = from_f<T>(acc * inv);
  }
}

template <typename T>
int launch_attention_generic(const T* qkv, T* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                             cudaStream_t st) {
  int maxkeys;
  if (attn_type == KDB_ATTN_GLOBAL) {
    maxkeys = h * w;
  } else if (attn_type == KDB_ATTN_NEIGHBORHOOD) {
    KDB_REQUIRE(attn_param >= 1 && h >= attn_param && w >= attn_param, KDB_ERR_BAD_SHAPE,
                "neighborhood attention: grid %dx%d smaller than kernel %d", h, w, attn_param);
    maxkeys = attn_param * attn_param;
  } else if (attn_type == KDB_ATTN_SHIFTED_WINDOW) {
    KDB_REQUIRE(attn_param >= 1 && h % attn_param == 0 && w % attn_param == 0, KDB_ERR_BAD_SHAPE,
                "shifted-window attention: grid %dx%d not divisible by window %d", h, w, attn_param);
    maxkeys = attn_param * attn_param;
  } else {
    KDB_REQUIRE(false, KDB_ERR_BAD_ARG, "attention: bad type %d", attn_type);
  }
  const size_t smem = sizeof(float) * 4 * (size_t)(e + 2 * maxkeys);
  KDB_REQUIRE(smem <= 200 * 1024, KDB_ERR_UNSUPPORTED, "attention_generic: %d keys exceed the shared-memory budget", maxkeys);
  static bool attr_f = false, attr_b = false;
  bool& attr = std::is_same<T, float>::value ? attr_f : attr_b;
  if (!attr) {
    KDB_CUDA(cudaFuncSetAttribute(attn_generic_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  dim3 grid((unsigned)ceil_div(h * w, 4), (unsigned)nh, (unsigned)B);
  attn_generic_kernel<T><<<grid, 128, smem, st>>>(qkv, out, h, w, nh, e, attn_type, attn_param, shift, maxkeys);
  KDB_LAUNCH_CHECK(F_ATTN_GENERIC, st);
  return 0;
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
    const float gelu = 0.5f * g * (1.f + erff(g * 0.70710678118654752440f));
    out[i] = from_f<T>(a * to_f(from_f<T>(gelu)));
  }
}

template <typename T>
int launch_geglu(const T* h, T* out, int64_t M, int F, cudaStream_t st) {
  int64_t blocks = ceil_div(M * F, 256);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  geglu_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(h, out, M, F);
  KDB_LAUNCH_CHECK(F_GEGLU, st);
  return 0;
}
template int launch_geglu<float>(const float*, float*, int64_t, int, cudaStream_t);
template int launch_geglu<bf16>(const bf16*, bf16*, int64_t, int, cudaStream_t);

template <typename T>
__global__ void __launch_bounds__(256) merge_gather_kernel(const T* __restrict__ x, T* __restrict__ out, int H, int Wd, int C,
                                                           int64_t total) {
  const int hc = H / 2, wc = Wd / 2;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int e = (int)(i % C);
    int64_t r = i / C;
    const int q = (int)(r & 3);
    r >>= 2;
    const int wx = (int)(r % wc);
    r /= wc;
    const int hy = (int)(r % hc);
    const int64_t b = r / hc;
    out[i] = x[((b * H + (2 * hy + (q >> 1))) * Wd + (2 * wx + (q & 1))) * C + e];
  }
}

template <typename T>
int launch_merge_gather(const T* x, T* out, int B, int H, int Wd, int C, cudaStream_t st) {
  KDB_REQUIRE(H % 2 == 0 && Wd % 2 == 0, KDB_ERR_BAD_SHAPE, "token merge: grid %dx%d not even", H, Wd);
  const int64_t total = (int64_t)B * H * Wd * C;
  int64_t blocks = ceil_div(total, 256);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  merge_gather_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(x, out, H, Wd, C, total);
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
  const int th_n = H / ph, tw_n = Wd / pw;
  const int64_t b = tok / ((int64_t)th_n * tw_n);
  const int r = (int)(tok - b * th_n * tw_n);
  const int ty = r / tw_n, tx = r - ty * tw_n;
  float c_skip = 0.f, c_out = 1.f, c_in;
  if (sd > 0.f) karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
  const int N = ph * pw * Cout;
  for (int n = lane; n < N; n += 32) {
    const float* wr = W + (int64_t)n * C0;
    float acc = 0.f;
    for (int k = 0; k < C0; ++k) acc = fmaf(xn[k], __ldg(wr + k), acc);
    acc = to_f(from_f<T>(acc));
    const int q = n / Cout, c = n - q * Cout;
    const int nh = q / pw, nw = q - nh * pw;
    const int64_t o = ((b * Cout + c) * H + (ty * ph + nh)) * Wd + (tx * pw + nw);
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

// y = x * scale * rsqrt(mean(x^2) + eps), vectors in shared memory
__device__ __forceinline__ void block_rmsnorm(const float* x, float* y, const float* __restrict__ scale, int n, float* red) {
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) ss = fmaf(x[i], x[i], ss);
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)n + kEps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = x[i] * (__ldg(scale + i) * rstd);
  __syncthreads();
}

__global__ void __launch_bounds__(256) conditioning_kernel(const CondWeights w, const float* __restrict__ sigma,
                                                           const float* __restrict__ aug, const int64_t* __restrict__ cls,
                                                           const float* __restrict__ mcond, float* __restrict__ out, int64_t out_stride) {
  extern __shared__ float4 cond_sm4[];          // 16-byte aligned: block_matvec reads its input vector as float4
  float* sm = reinterpret_cast<float*>(cond_sm4);
  const int mw = w.mw, dff = w.dff;
  float* ff = sm;              // [mw]   fourier features
  float* emb = ff + mw;        // [mw]   summed embedding / residual stream
  float* xn = emb + mw;        // [mw]
  float* up = xn + mw;         // [2*dff]
  float* red = up + 2 * dff;   // [32]
  float* mc = red + 32;        // [mcond_dim]
  const int row = blockIdx.x;
  const int half = mw / 2;
  const float two_pi = 6.283185307179586f;

  // time embedding: FourierFeatures(log(sigma)/4) -> time_in_proj        (:734-735, layers.py:291-293)
  const float c_noise = logf(sigma[row]) / 4.f;
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    const float f = (two_pi * c_noise) * __ldg(w.time_emb + j);
    float s, c;
    sincosf(f, &s, &c);
    ff[j] = c;
    ff[half + j] = s;
  }
  __syncthreads();
  block_matvec(w.time_in, ff, emb, 0, mw, mw, false);
  __syncthreads();
  // augmentation embedding (zeros when aug_cond is None, :736-737)
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    float f = 0.f;
    if (aug != nullptr)
      for (int k = 0; k < 9; ++k) f = fmaf(two_pi * aug[(int64_t)row * 9 + k], __ldg(w.aug_emb + j * 9 + k), f);
    float s, c;
    sincosf(f, &s, &c);
    ff[j] = c;
    ff[half + j] = s;
  }
  __syncthreads();
  block_matvec(w.aug_in, ff, emb, 0, mw, mw, true);
  __syncthreads();
  if (w.class_emb != nullptr) {
    const int64_t ci = cls[row];
    for (int j = threadIdx.x; j < mw; j += blockDim.x) emb[j] += __ldg(w.class_emb + ci * mw + j);
  }
  if (w.mcond_in != nullptr) {
    for (int j = threadIdx.x; j < w.mcond_dim; j += blockDim.x) mc[j] = mcond[(int64_t)row * w.mcond_dim + j];
    __syncthreads();
    block_matvec(w.mcond_in, mc, emb, 0, mw, w.mcond_dim, true);
  }
  __syncthreads();

  // MappingNetwork (:569-581)
  block_rmsnorm(emb, emb, w.in_norm, mw, red);
  for (int l = 0; l < w.depth; ++l) {
    block_rmsnorm(emb, xn, w.blk_norm[l], mw, red);
    block_matvec(w.blk_up[l], xn, up, 0, 2 * dff, mw, false);
    __syncthreads();
    for (int i = threadIdx.x; i < dff; i += blockDim.x) {
      const float g = up[dff + i];
      up[i] = up[i] * (0.5f * g * (1.f + erff(g * 0.70710678118654752440f)));
    }
    __syncthreads();
    block_matvec(w.blk_down[l], up, emb, 0, mw, dff, true);
    __syncthreads();
  }
  block_rmsnorm(emb, xn, w.out_norm, mw, red);

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

// ------------------------------------------------------------------------------------------------
// dtype conversion
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) out[i] = __float2bfloat16_rn(in[i]);
}
int launch_f32_to_bf16(const float* in, bf16* out, int64_t n, cudaStream_t st) {
  int64_t blocks = ceil_div(n, 256);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  f32_to_bf16_kernel<<<(unsigned)blocks, 256, 0, st>>>(in, out, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

template <typename T>
__global__ void __launch_bounds__(256) to_f32_kernel(const T* __restrict__ in, float* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) out[i] = to_f(in[i]);
}
template <typename T>
int launch_to_f32(const T* in, float* out, int64_t n, cudaStream_t st) {
  int64_t blocks = ceil_div(n, 256);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  to_f32_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(in, out, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}
template int launch_to_f32<float>(const float*, float*, int64_t, cudaStream_t);
template int launch_to_f32<bf16>(const bf16*, float*, int64_t, cudaStream_t);

}  // namespace kdb
