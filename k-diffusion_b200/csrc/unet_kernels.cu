// unet_kernels.cu -- fp32 kernels of the image_v1 U-Net engine (unet_engine.cu).  Token-major activations [B, H, W, C].
#include <cmath>

#include "simt_tile.cuh"
#include "unet_kernels.cuh"

namespace kdb {

namespace {

constexpr float kGnEps = 1e-5f;                 // AdaGN eps (layers.py:163)

// ------------------------------------------------------------------------------------------------
// implicit-GEMM convolution on the SIMT GEMM's tile loop (simt_tile.cuh), A gathered per tap
// ------------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(256) unet_conv_kernel(const ConvArgs a) {
  const int64_t M = (int64_t)a.B * a.H * a.W;
  const int Ct = a.c1 + a.c2, K = KS * KS * Ct, N = a.N;
  const int64_t m0 = (int64_t)blockIdx.y * kTileM;
  const int n0 = blockIdx.x * kTileN;
  const int tid = threadIdx.x;
  const int lr = tid >> 2, lk = (tid & 3) * 4;   // loader: row 0..63, k offset 0,4,8,12
  // pixel of the A row this thread loads
  const int64_t am = m0 + lr;
  const bool arow = am < M;
  int ay = 0, ax = 0;
  if (arow) {
    const int r = (int)(am % ((int64_t)a.H * a.W));
    ay = r / a.W;
    ax = r - ay * a.W;
  }
  auto fill = [&](int k0, TileSmem& As, TileSmem& Ws) {
    const int k = k0 + lk;
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f), wv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (arow && k < K) {
      const int tap = k / Ct, c = k - tap * Ct;
      const int yy = ay + tap / KS - KS / 2, xx = ax + tap % KS - KS / 2;
      if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W) {
        const int64_t pix = am + (int64_t)(tap / KS - KS / 2) * a.W + (tap % KS - KS / 2);   // same image: the row is in bounds
        const float* src = c < a.c1 ? a.in1 + pix * a.c1 + c : a.in2 + pix * a.c2 + (c - a.c1);
        av = *reinterpret_cast<const float4*>(src);
      }
    }
    if (n0 + lr < N && k < K) wv = __ldg(reinterpret_cast<const float4*>(a.w + (int64_t)(n0 + lr) * K + k));
    As[lk + 0][lr] = av.x; As[lk + 1][lr] = av.y; As[lk + 2][lr] = av.z; As[lk + 3][lr] = av.w;
    Ws[lk + 0][lr] = wv.x; Ws[lk + 1][lr] = wv.y; Ws[lk + 2][lr] = wv.z; Ws[lk + 3][lr] = wv.w;
  };
  simt_tile(m0, n0, M, N, K, fill, [&](int64_t m, int n, float v) {
    if (a.bias != nullptr) v += __ldg(a.bias + n);
    if (a.r1 != nullptr) v += n < a.rc1 ? a.r1[m * a.rc1 + n] : a.r2[m * (N - a.rc1) + (n - a.rc1)];
    a.out[m * N + n] = v;
  });
}

// ------------------------------------------------------------------------------------------------
// AdaGN (+ GELU): one CTA per (group, image)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) unet_adagn_kernel(const float* __restrict__ in1, int c1, const float* __restrict__ in2, int c2,
                                                         float* __restrict__ out, const float* __restrict__ cond, int64_t cond_bs, int ada_off,
                                                         int groups, int gelu, int HW) {
  __shared__ float red[32];
  const int g = blockIdx.x, b = blockIdx.y;
  const int C = c1 + c2, cg = C / groups;
  const int64_t n = (int64_t)HW * cg;
  const int64_t pix0 = (int64_t)b * HW;
  auto load = [&](int64_t i, int& c, int64_t& pix) {
    const int64_t p = i / cg;
    c = g * cg + (int)(i - p * cg);
    pix = pix0 + p;
    return c < c1 ? in1[pix * c1 + c] : in2[pix * c2 + (c - c1)];
  };
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    s += load(i, c, pix);
  }
  const float mean = block_sum(s, red) / (float)n;
  float q = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    const float d = load(i, c, pix) - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)n + kGnEps);
  const float* row = cond + (int64_t)b * cond_bs + ada_off;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    const float v = (load(i, c, pix) - mean) * rstd;
    float y = fmaf(v, __ldg(row + c) + 1.f, __ldg(row + C + c));
    if (gelu) y = gelu_erf(y);
    out[pix * C + c] = y;
  }
}

// ------------------------------------------------------------------------------------------------
// 2x resampling with reflect padding
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect1(int p, int n) { return p < 0 ? -p : (p >= n ? 2 * n - 2 - p : p); }

__global__ void __launch_bounds__(256) unet_down_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)B * Ho * Wo * C;
  const float k[4] = {0.125f, 0.375f, 0.375f, 0.125f};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t t = i / C;
    int b, oy, ox;
    token_coords(t, Ho, Wo, b, oy, ox);
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int yy = reflect1(2 * oy + u - 1, H);
      float r = 0.f;
#pragma unroll
      for (int v = 0; v < 4; ++v) r = fmaf(k[v], in[(((int64_t)b * H + yy) * W + reflect1(2 * ox + v - 1, W)) * C + c], r);
      acc = fmaf(k[u], r, acc);
    }
    out[i] = acc;
  }
}

// conv_transpose2d(reflect_pad(x, 1), 2 * [1,3,3,1]/8 outer product, stride 2, padding 3): output row 2m takes x rows m (3/4) and
// m - 1 (1/4), row 2m + 1 takes rows m (3/4) and m + 1 (1/4), reflected at the border; the same along columns
__global__ void __launch_bounds__(256) unet_up_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C) {
  const int Ho = 2 * H, Wo = 2 * W;
  const int64_t total = (int64_t)B * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t t = i / C;
    int b, oy, ox;
    token_coords(t, Ho, Wo, b, oy, ox);
    const int my = oy >> 1, mx = ox >> 1;
    const int ys[2] = {my, reflect1((oy & 1) ? my + 1 : my - 1, H)};
    const int xs[2] = {mx, reflect1((ox & 1) ? mx + 1 : mx - 1, W)};
    const float k[2] = {0.75f, 0.25f};
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      float r = 0.f;
#pragma unroll
      for (int v = 0; v < 2; ++v) r = fmaf(k[v], in[(((int64_t)b * H + ys[u]) * W + xs[v]) * C + c], r);
      acc = fmaf(k[u], r, acc);
    }
    out[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// patch-in / patch-out
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) unet_patch_in_kernel(const float* __restrict__ x, const float* __restrict__ sigma, float sd,
                                                            const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out,
                                                            int B, int Cin, int H, int W, int p, int N) {
  const int h = H / p, wd = W / p, Kin = Cin * p * p;
  const int64_t total = (int64_t)B * h * wd * N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int o = (int)(i % N);
    int b, ty, tx;
    token_coords(i / N, h, wd, b, ty, tx);
    float c_skip, c_out, c_in = 1.f;
    if (sd > 0.f) karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
    float acc = 0.f;
    for (int k = 0; k < Kin; ++k) {   // pixel_unshuffle channel k = (c, i, j)
      const int c = k / (p * p), r = k - c * p * p;
      const float v = x[nchw_offset(b, c, ty * p + r / p, tx * p + r % p, Cin, H, W)] * c_in;
      acc = fmaf(__ldg(w + (int64_t)o * Kin + k), v, acc);
    }
    out[i] = acc + __ldg(bias + o);
  }
}

__global__ void __launch_bounds__(256) unet_patch_out_kernel(const float* __restrict__ tok, const float* __restrict__ w,
                                                             const float* __restrict__ bias, const float* __restrict__ x_in,
                                                             const float* __restrict__ sigma, float sd, float* __restrict__ out, int B, int Cout,
                                                             int H, int W, int p, int K) {
  const int64_t total = (int64_t)B * Cout * H * W;
  const int wd = W / p;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int c = (int)((i / ((int64_t)W * H)) % Cout);
    const int b = (int)(i / ((int64_t)W * H * Cout));
    const int o = (c * p + y % p) * p + x % p;                   // pixel_shuffle: channel (c, i, j) -> pixel (y*p + i, x*p + j)
    const float* t = tok + (((int64_t)b * (H / p) + y / p) * wd + x / p) * K;
    const float* wr = w + (int64_t)o * K;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(__ldg(wr + k), t[k], acc);
    float f = acc + __ldg(bias + o);
    if (sd > 0.f) {
      float c_skip, c_out, c_in;
      karras_scalings(sigma[b], sd, c_skip, c_out, c_in);
      f = f * c_out + x_in[i] * c_skip;
    }
    out[i] = f;
  }
}

// proj_out's variance row averaged over the token grid (image_v1.py:151-152), one CTA per image: each thread forms w_v . y[b, t] for the
// tokens t = threadIdx.x (mod 256) in order, then a fixed-order block sum
__global__ void __launch_bounds__(256) unet_logvar_kernel(const float* __restrict__ tok, const float* __restrict__ wv, const float* __restrict__ bv,
                                                          float* __restrict__ logvar, int T, int K) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float acc = 0.f;
  for (int t = threadIdx.x; t < T; t += 256) {
    const float* y = tok + ((int64_t)b * T + t) * K;
    float d = 0.f;
    for (int k = 0; k < K; ++k) d = fmaf(__ldg(wv + k), y[k], d);
    acc = __fadd_rn(acc, d);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) logvar[b] = __fadd_rn(__ldg(bv), __fdiv_rn(acc, (float)T));
}

// ------------------------------------------------------------------------------------------------
// conditioning
// ------------------------------------------------------------------------------------------------
// vout[o] = bias[o] + W[o, :] . vin for o in [o_begin, o_end): one warp per output, lanes over the inputs in a fixed order
__device__ __forceinline__ void warp_matvec(const float* __restrict__ W, const float* __restrict__ bias, const float* vin, float* vout,
                                            int o_begin, int o_end, int n_in, bool gelu) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int o = o_begin + warp; o < o_end; o += nw) {
    const float* wr = W + (int64_t)o * n_in;
    float s = 0.f;
    for (int k = lane; k < n_in; k += 32) s = fmaf(__ldg(wr + k), vin[k], s);
    s = warp_sum(s);
    if (lane == 0) {
      float v = s + (bias ? __ldg(bias + o) : 0.f);
      vout[o] = gelu ? gelu_erf(v) : v;
    }
  }
}

__global__ void __launch_bounds__(256) unet_cond_kernel(const UNetCondWeights w, const float* __restrict__ sigma, const float* __restrict__ aug,
                                                        const float* __restrict__ mcond, float* __restrict__ out, int64_t out_stride) {
  extern __shared__ float usm[];
  const int mw = w.mw, half = mw / 2, row = blockIdx.x;
  float* h = usm;             // [mw]
  float* h2 = h + mw;         // [mw]
  float* v = h2 + mw;         // [mcond_dim]
  const float c_noise = logf(sigma[row]) / 4.f;
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    float s, c;
    sincosf(6.283185307179586f * c_noise * __ldg(w.time_emb + j), &s, &c);
    h[j] = c;
    h[half + j] = s;
  }
  // mapping_cond vector: [aug_cond or zeros(9), mapping_cond] with the augment wrapper, else mapping_cond (NULL: no term)
  const bool has_mc = w.mcond_dim > 0 && (w.augment || mcond != nullptr);
  if (has_mc) {
    const int na = w.augment ? 9 : 0;
    for (int k = threadIdx.x; k < w.mcond_dim; k += blockDim.x)
      v[k] = k < na ? (aug ? aug[(int64_t)row * 9 + k] : 0.f) : mcond[(int64_t)row * (w.mcond_dim - na) + (k - na)];
  }
  __syncthreads();
  if (has_mc) {
    warp_matvec(w.mcond_w, nullptr, v, h2, 0, mw, w.mcond_dim, false);
    __syncthreads();
    for (int j = threadIdx.x; j < mw; j += blockDim.x) h[j] += h2[j];
  }
  __syncthreads();
  warp_matvec(w.map_w0, w.map_b0, h, h2, 0, mw, mw, true);      // MappingNet (image_v1.py:80-86)
  __syncthreads();
  warp_matvec(w.map_w1, w.map_b1, h2, h, 0, mw, mw, true);
  __syncthreads();
  // every AdaGN mapper; the CTAs of one row (gridDim.y) share the outputs and each repeats the short mapping network
  float* orow = out + (int64_t)row * out_stride;
  const int per = (w.ada_total + (int)gridDim.y - 1) / (int)gridDim.y;
  const int o0 = (int)blockIdx.y * per, o1 = min(w.ada_total, o0 + per);
  warp_matvec(w.ada_w, w.ada_b, h, orow, o0, o1, mw, false);
  if (blockIdx.y == 0)
    for (int j = threadIdx.x; j < mw; j += blockDim.x) orow[w.ada_total + j] = h[j];
}

__global__ void __launch_bounds__(256) unet_reorder_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int C, int kk,
                                                           int scaled_rows, float scale) {
  const int64_t total = (int64_t)N * C * kk;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % kk);
    const int c = (int)((i / kk) % C);
    const int64_t n = i / ((int64_t)kk * C);
    const float v = src[i];
    dst[(n * kk + t) * C + c] = n < scaled_rows ? v * scale : v;
  }
}

unsigned grid_for(int64_t n) { return (unsigned)std::min<int64_t>(ceil_div(n, 256), (int64_t)kNumSMs * 32); }

// ------------------------------------------------------------------------------------------------
// backward (training) kernels
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_slope(float y) {   // d gelu_erf / dy = Phi(y) + y phi(y)
  const float Phi = 0.5f * (1.f + erff(y * kRsqrt2));
  return fmaf(y, 0.39894228040143267794f * expf(-0.5f * y * y), Phi);
}

// AdaGN (+ GELU) backward: one CTA per (group, image), mean and rstd recomputed in unet_adagn_kernel's order.  Per channel of the group,
// d scale = sum_p dy' x^ and d shift = sum_p dy' (dy' = dy gelu'(y) with GELU) by one warp each over the pixels; then
// dx = rstd ((1 + scale) dy' - mean_g((1 + scale) dy') - x^ mean_g((1 + scale) dy' x^)) [+ add], written to the source it was read from.
__global__ void __launch_bounds__(256) unet_adagn_vjp_kernel(const float* __restrict__ in1, int c1, const float* __restrict__ in2, int c2,
                                                             const float* __restrict__ dy, const float* add, float* out1, float* out2,
                                                             const float* __restrict__ cond, int64_t cond_bs, int ada_off, float* __restrict__ dss,
                                                             int64_t dss_bs, int groups, int gelu, int HW) {
  extern __shared__ float chs[];                 // [cg] d scale, [cg] d shift
  __shared__ float red[32];
  const int g = blockIdx.x, b = blockIdx.y;
  const int C = c1 + c2, cg = C / groups;
  const int64_t n = (int64_t)HW * cg;
  const int64_t pix0 = (int64_t)b * HW;
  auto at = [&](int64_t pix, int c) { return c < c1 ? in1[pix * c1 + c] : in2[pix * c2 + (c - c1)]; };
  auto load = [&](int64_t i, int& c, int64_t& pix) {
    const int64_t p = i / cg;
    c = g * cg + (int)(i - p * cg);
    pix = pix0 + p;
    return at(pix, c);
  };
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    s += load(i, c, pix);
  }
  const float mean = block_sum(s, red) / (float)n;
  float q = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    const float d = load(i, c, pix) - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)n + kGnEps);
  const float* row = cond + (int64_t)b * cond_bs + ada_off;
  auto grad_y = [&](float v, int64_t pix, int c) {   // the gradient at the AdaGN output, through the GELU
    const float d = dy[pix * C + c];
    return gelu ? d * gelu_slope(fmaf(v, __ldg(row + c) + 1.f, __ldg(row + C + c))) : d;
  };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int cl = warp; cl < cg; cl += nw) {
    const int c = g * cg + cl;
    float ds = 0.f, dt = 0.f;
    for (int p = lane; p < HW; p += 32) {
      const float v = (at(pix0 + p, c) - mean) * rstd, d = grad_y(v, pix0 + p, c);
      ds = fmaf(d, v, ds);
      dt += d;
    }
    ds = warp_sum(ds);
    dt = warp_sum(dt);
    if (lane == 0) chs[cl] = ds, chs[cg + cl] = dt;
  }
  __syncthreads();
  float sa = 0.f, sb = 0.f;
  for (int cl = 0; cl < cg; ++cl) {
    const float sc = __ldg(row + g * cg + cl) + 1.f;
    sa = fmaf(sc, chs[cg + cl], sa);
    sb = fmaf(sc, chs[cl], sb);
  }
  sa /= (float)n;
  sb /= (float)n;
  float* drow = dss + (int64_t)b * dss_bs + ada_off;
  for (int cl = threadIdx.x; cl < cg; cl += blockDim.x) {
    drow[g * cg + cl] = chs[cl];
    drow[C + g * cg + cl] = chs[cg + cl];
  }
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    int c;
    int64_t pix;
    const float v = (load(i, c, pix) - mean) * rstd;
    float dx = rstd * (grad_y(v, pix, c) * (__ldg(row + c) + 1.f) - sa - v * sb);
    if (add != nullptr) dx += add[pix * C + c];
    if (c < c1)
      out1[pix * c1 + c] = dx;
    else
      out2[pix * c2 + (c - c1)] = dx;
  }
}

// the weight with which input row y of a grid of H rows enters output row o of the 2x resampling (reflect padding included)
__device__ __forceinline__ float down_weight(int o, int y, int H) {
  const float k[4] = {0.125f, 0.375f, 0.375f, 0.125f};
  float w = 0.f;
#pragma unroll
  for (int u = 0; u < 4; ++u) w += reflect1(2 * o + u - 1, H) == y ? k[u] : 0.f;
  return w;
}
__device__ __forceinline__ float up_weight(int o, int y, int H) {
  const int m = o >> 1;
  return (m == y ? 0.75f : 0.f) + (reflect1((o & 1) ? m + 1 : m - 1, H) == y ? 0.25f : 0.f);
}

// Resampling adjoint in gather form: one thread per input element (b, y, x, c) sums every output element that read it, with the product of
// its row and column weights; the output rows that can reach row y lie within a few rows of y / 2 (down) or 2 y (up), reflections included.
template <bool UP>
__global__ void __launch_bounds__(256) unet_resample_vjp_kernel(const float* __restrict__ dout, const float* add, float* din, int B, int H, int W,
                                                                int C) {
  const int Ho = UP ? 2 * H : H / 2, Wo = UP ? 2 * W : W / 2;
  const int64_t total = (int64_t)B * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int b, y, x;
    token_coords(i / C, H, W, b, y, x);
    const int oy0 = max(0, UP ? 2 * y - 3 : y / 2 - 2), oy1 = min(Ho - 1, UP ? 2 * y + 4 : y / 2 + 2);
    const int ox0 = max(0, UP ? 2 * x - 3 : x / 2 - 2), ox1 = min(Wo - 1, UP ? 2 * x + 4 : x / 2 + 2);
    float acc = 0.f;
    for (int oy = oy0; oy <= oy1; ++oy) {
      const float wy = UP ? up_weight(oy, y, H) : down_weight(oy, y, H);
      if (wy == 0.f) continue;
      float r = 0.f;
      for (int ox = ox0; ox <= ox1; ++ox) {
        const float wx = UP ? up_weight(ox, x, W) : down_weight(ox, x, W);
        if (wx != 0.f) r = fmaf(wx, dout[(((int64_t)b * Ho + oy) * Wo + ox) * C + c], r);
      }
      acc = fmaf(wy, r, acc);
    }
    din[i] = add != nullptr ? acc + add[i] : acc;
  }
}

// tap-major [N, kk, C] -> the tap-major weight of the input-gradient convolution [C, kk, N], taps reversed
__global__ void __launch_bounds__(256) unet_flip_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int C, int kk) {
  const int64_t total = (int64_t)N * C * kk;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i % N);
    const int t = (int)((i / N) % kk);
    const int64_t c = i / ((int64_t)N * kk);
    dst[i] = src[((int64_t)n * kk + (kk - 1 - t)) * C + c];
  }
}

// pixel_unshuffle of NCHW x [B, C, H, W] to token rows [B (H/p) (W/p), ld], column (c, i, j); column C p p holds col[b] / (h w) when col is
// given, every other column past C p p zero
__global__ void __launch_bounds__(256) unet_unshuffle_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int C, int H, int W, int p,
                                                             int ld, const float* __restrict__ col) {
  const int h = H / p, wd = W / p, K = C * p * p;
  const int64_t total = (int64_t)B * h * wd * ld;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int o = (int)(i % ld);
    float v = 0.f;
    if (o < K) {
      int b, ty, tx;
      token_coords(i / ld, h, wd, b, ty, tx);
      const int c = o / (p * p), r = o - c * p * p;
      v = x[nchw_offset(b, c, ty * p + r / p, tx * p + r % p, C, H, W)];
    } else if (o == K && col != nullptr) {
      v = __fdiv_rn(col[i / ld / ((int64_t)h * wd)], (float)(h * wd));
    }
    out[i] = v;
  }
}

// out[m, k] = sum_{o < N} U[m, o] W[o, k]: proj_out's input gradient (N = its few output channels)
__global__ void __launch_bounds__(256) unet_proj_out_vjp_kernel(const float* __restrict__ U, const float* __restrict__ Wt, float* __restrict__ out,
                                                                int64_t M, int N, int K) {
  const int64_t total = M * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / K;
    const int k = (int)(i - m * K);
    float acc = 0.f;
    for (int o = 0; o < N; ++o) acc = fmaf(U[m * N + o], __ldg(Wt + (int64_t)o * K + k), acc);
    out[i] = acc;
  }
}

__global__ void __launch_bounds__(256) unet_scale_kernel(float* p, int64_t n, float s) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] *= s;
}

// The mapping network's backward, one CTA per row: recomputes unet_cond_kernel's h0 = FourierFeatures + mapping_cond Linear, z0 = W0 h0 + b0,
// a0 = gelu(z0), z1 = W1 a0 + b1 in its order; from dcond (the gradient of gelu(z1)) writes dz1, dz0 and dh0 = W0^T dz0, and keeps h0, a0
// and the mapping_cond vector v for the weight gradients.
__global__ void __launch_bounds__(256) unet_mapping_vjp_kernel(const UNetCondWeights w, const float* __restrict__ sigma, const float* __restrict__ aug,
                                                               const float* __restrict__ mcond, const float* __restrict__ dcond, UNetMapGrad o) {
  extern __shared__ float usm[];
  const int mw = w.mw, half = mw / 2, row = blockIdx.x, mcd = w.mcond_dim;
  float* h = usm;
  float* z0 = h + mw;
  float* a0 = z0 + mw;
  float* z1 = a0 + mw;
  float* d1 = z1 + mw;
  float* d0 = d1 + mw;
  float* v = d0 + mw;     // [mcond_dim]
  const float c_noise = logf(sigma[row]) / 4.f;
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    float s, c;
    sincosf(6.283185307179586f * c_noise * __ldg(w.time_emb + j), &s, &c);
    h[j] = c;
    h[half + j] = s;
  }
  const bool has_mc = mcd > 0 && (w.augment || mcond != nullptr);
  const int na = w.augment ? 9 : 0;
  for (int k = threadIdx.x; k < mcd; k += blockDim.x)
    v[k] = !has_mc ? 0.f : k < na ? (aug ? aug[(int64_t)row * 9 + k] : 0.f) : mcond[(int64_t)row * (mcd - na) + (k - na)];
  __syncthreads();
  if (has_mc) {
    warp_matvec(w.mcond_w, nullptr, v, z0, 0, mw, mcd, false);
    __syncthreads();
    for (int j = threadIdx.x; j < mw; j += blockDim.x) h[j] += z0[j];
  }
  __syncthreads();
  warp_matvec(w.map_w0, w.map_b0, h, z0, 0, mw, mw, false);
  __syncthreads();
  for (int j = threadIdx.x; j < mw; j += blockDim.x) a0[j] = gelu_erf(z0[j]);
  __syncthreads();
  warp_matvec(w.map_w1, w.map_b1, a0, z1, 0, mw, mw, false);
  __syncthreads();
  for (int j = threadIdx.x; j < mw; j += blockDim.x) d1[j] = dcond[(int64_t)row * mw + j] * gelu_slope(z1[j]);
  __syncthreads();
  for (int k = threadIdx.x; k < mw; k += blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < mw; ++j) s = fmaf(__ldg(w.map_w1 + (int64_t)j * mw + k), d1[j], s);
    d0[k] = s * gelu_slope(z0[k]);
  }
  __syncthreads();
  const int64_t r = (int64_t)row * mw;
  for (int k = threadIdx.x; k < mw; k += blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < mw; ++j) s = fmaf(__ldg(w.map_w0 + (int64_t)j * mw + k), d0[j], s);
    o.dh0[r + k] = s;
    o.h0[r + k] = h[k];
    o.a0[r + k] = a0[k];
    o.dz0[r + k] = d0[k];
    o.dz1[r + k] = d1[k];
  }
  for (int k = threadIdx.x; k < mcd; k += blockDim.x) o.v[(int64_t)row * mcd + k] = v[k];
}

}  // namespace

int launch_unet_conv(const ConvArgs& a, int ks, cudaStream_t st) {
  KDB_REQUIRE(ks == 1 || ks == 3, KDB_ERR_BAD_ARG, "unet_conv: kernel size %d", ks);
  KDB_REQUIRE(a.in1 && a.w && a.out && a.B > 0 && a.H > 0 && a.W > 0 && a.N > 0 && a.c1 > 0, KDB_ERR_BAD_ARG, "unet_conv: bad arguments");
  KDB_REQUIRE(a.c1 % 4 == 0 && a.c2 % 4 == 0 && (a.c2 == 0 || a.in2) && a.rc1 % 4 == 0, KDB_ERR_BAD_SHAPE,
              "unet_conv: channel counts %d + %d must be multiples of 4", a.c1, a.c2);
  KDB_REQUIRE(!a.r1 || a.rc1 == a.N || (a.r2 && a.rc1 < a.N), KDB_ERR_BAD_ARG, "unet_conv: bad residual split");
  const int64_t M = (int64_t)a.B * a.H * a.W;
  dim3 grid((unsigned)ceil_div(a.N, kTileN), (unsigned)ceil_div(M, kTileM));
  KDB_REQUIRE(grid.y <= 65535u, KDB_ERR_BAD_SHAPE, "unet_conv: %lld pixels exceed the grid", (long long)M);
  if (ks == 3)
    unet_conv_kernel<3><<<grid, 256, 0, st>>>(a);
  else
    unet_conv_kernel<1><<<grid, 256, 0, st>>>(a);
  KDB_LAUNCH_CHECK(F_UNET_CONV, st);
  return 0;
}

int launch_unet_adagn(const float* in1, int c1, const float* in2, int c2, float* out, const float* cond, int64_t cond_bs, int ada_off, int groups,
                      bool gelu, int B, int HW, cudaStream_t st) {
  KDB_REQUIRE(groups >= 1 && (c1 + c2) % groups == 0 && (c2 == 0 || in2), KDB_ERR_BAD_SHAPE, "unet_adagn: %d channels in %d groups", c1 + c2,
              groups);
  unet_adagn_kernel<<<dim3((unsigned)groups, (unsigned)B), 256, 0, st>>>(in1, c1, in2, c2, out, cond, cond_bs, ada_off, groups, gelu ? 1 : 0, HW);
  KDB_LAUNCH_CHECK(F_UNET_ADAGN, st);
  return 0;
}

int launch_unet_resample(const float* in, float* out, int B, int H, int W, int C, bool up, cudaStream_t st) {
  KDB_REQUIRE(H >= 2 && W >= 2, KDB_ERR_BAD_SHAPE, "unet_resample: grid %dx%d too small for reflect padding", H, W);
  const int64_t total = (int64_t)B * C * (up ? 4LL * H * W : (int64_t)(H / 2) * (W / 2));
  if (up)
    unet_up_kernel<<<grid_for(total), 256, 0, st>>>(in, out, B, H, W, C);
  else
    unet_down_kernel<<<grid_for(total), 256, 0, st>>>(in, out, B, H, W, C);
  KDB_LAUNCH_CHECK(F_UNET_RESAMPLE, st);
  return 0;
}

int launch_unet_patch_in(const float* x, const float* sigma, float sigma_data, const float* w, const float* bias, float* out, int B, int Cin,
                         int H, int W, int p, int N, cudaStream_t st) {
  unet_patch_in_kernel<<<grid_for((int64_t)B * (H / p) * (W / p) * N), 256, 0, st>>>(x, sigma, sigma_data, w, bias, out, B, Cin, H, W, p, N);
  KDB_LAUNCH_CHECK(F_UNET_PATCH, st);
  return 0;
}

int launch_unet_patch_out(const float* tokens, const float* w, const float* bias, const float* x_in, const float* sigma, float sigma_data,
                          float* out, int B, int Cout, int H, int W, int p, int K, cudaStream_t st) {
  unet_patch_out_kernel<<<grid_for((int64_t)B * Cout * H * W), 256, 0, st>>>(tokens, w, bias, x_in, sigma, sigma_data, out, B, Cout, H, W, p, K);
  KDB_LAUNCH_CHECK(F_UNET_PATCH, st);
  return 0;
}

int launch_unet_logvar(const float* tokens, const float* wv, const float* bv, float* logvar, int B, int T, int K, cudaStream_t st) {
  KDB_REQUIRE(tokens && wv && bv && logvar && B > 0 && T > 0 && K > 0, KDB_ERR_BAD_ARG, "unet_logvar: bad arguments");
  unet_logvar_kernel<<<(unsigned)B, 256, 0, st>>>(tokens, wv, bv, logvar, T, K);
  KDB_LAUNCH_CHECK(F_UNET_PATCH, st);
  return 0;
}

int launch_unet_conditioning(const UNetCondWeights& w, int rows, const float* sigma, const float* aug, const float* mcond, float* out,
                             int64_t out_stride, cudaStream_t st) {
  KDB_REQUIRE(w.mw % 2 == 0 && w.mw > 0, KDB_ERR_UNSUPPORTED, "unet_conditioning: mapping_out must be even");
  const size_t smem = sizeof(float) * (size_t)(2 * w.mw + w.mcond_dim);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "unet_conditioning: mapping network too wide");
  unet_cond_kernel<<<dim3((unsigned)rows, 4), 256, smem, st>>>(w, sigma, aug, mcond, out, out_stride);
  KDB_LAUNCH_CHECK(F_UNET_COND, st);
  return 0;
}

int launch_unet_reorder_conv_weight(const float* src, float* dst, int N, int C, int ks, int scaled_rows, float scale, cudaStream_t st) {
  unet_reorder_kernel<<<grid_for((int64_t)N * C * ks * ks), 256, 0, st>>>(src, dst, N, C, ks * ks, scaled_rows, scale);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

int launch_unet_adagn_vjp(const float* in1, int c1, const float* in2, int c2, const float* dy, const float* add, float* out1, float* out2,
                          const float* cond, int64_t cond_bs, int ada_off, float* dss, int64_t dss_bs, int groups, bool gelu, int B, int HW,
                          cudaStream_t st) {
  KDB_REQUIRE(groups >= 1 && (c1 + c2) % groups == 0 && (c2 == 0 || (in2 && out2)) && B > 0 && HW > 0, KDB_ERR_BAD_SHAPE,
              "unet_adagn_vjp: %d channels in %d groups", c1 + c2, groups);
  const size_t smem = sizeof(float) * 2 * ((c1 + c2) / groups);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "unet_adagn_vjp: %d channels per group", (c1 + c2) / groups);
  unet_adagn_vjp_kernel<<<dim3((unsigned)groups, (unsigned)B), 256, smem, st>>>(in1, c1, in2, c2, dy, add, out1, out2, cond, cond_bs, ada_off, dss,
                                                                                 dss_bs, groups, gelu ? 1 : 0, HW);
  KDB_LAUNCH_CHECK(F_UNET_ADAGN, st);
  return 0;
}

int launch_unet_resample_vjp(const float* dout, const float* add, float* din, int B, int H, int W, int C, bool up, cudaStream_t st) {
  KDB_REQUIRE(H >= 2 && W >= 2 && B > 0 && C > 0, KDB_ERR_BAD_SHAPE, "unet_resample_vjp: grid %dx%d too small for reflect padding", H, W);
  const int64_t total = (int64_t)B * H * W * C;
  if (up)
    unet_resample_vjp_kernel<true><<<grid_for(total), 256, 0, st>>>(dout, add, din, B, H, W, C);
  else
    unet_resample_vjp_kernel<false><<<grid_for(total), 256, 0, st>>>(dout, add, din, B, H, W, C);
  KDB_LAUNCH_CHECK(F_UNET_RESAMPLE, st);
  return 0;
}

int launch_unet_flip_conv_weight(const float* src, float* dst, int N, int C, int ks, cudaStream_t st) {
  unet_flip_kernel<<<grid_for((int64_t)N * C * ks * ks), 256, 0, st>>>(src, dst, N, C, ks * ks);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

int launch_unet_unshuffle(const float* x, float* out, int B, int C, int H, int W, int p, int ld, const float* col, cudaStream_t st) {
  KDB_REQUIRE(col == nullptr || ld > C * p * p, KDB_ERR_BAD_ARG, "unet_unshuffle: no column %d for the per-image value in rows of %d", C * p * p,
              ld);
  unet_unshuffle_kernel<<<grid_for((int64_t)B * (H / p) * (W / p) * ld), 256, 0, st>>>(x, out, B, C, H, W, p, ld, col);
  KDB_LAUNCH_CHECK(F_UNET_PATCH, st);
  return 0;
}

int launch_unet_proj_out_vjp(const float* U, const float* w, float* out, int64_t M, int N, int K, cudaStream_t st) {
  unet_proj_out_vjp_kernel<<<grid_for(M * K), 256, 0, st>>>(U, w, out, M, N, K);
  KDB_LAUNCH_CHECK(F_UNET_PATCH, st);
  return 0;
}

int launch_unet_scale(float* p, int64_t n, float s, cudaStream_t st) {
  if (p == nullptr || n <= 0) return 0;
  unet_scale_kernel<<<grid_for(n), 256, 0, st>>>(p, n, s);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

int launch_unet_mapping_vjp(const UNetCondWeights& w, int rows, const float* sigma, const float* aug, const float* mcond, const float* dcond,
                            const UNetMapGrad& out, cudaStream_t st) {
  const size_t smem = sizeof(float) * (size_t)(6 * w.mw + w.mcond_dim);
  KDB_REQUIRE(smem <= 48 * 1024, KDB_ERR_UNSUPPORTED, "unet_mapping_vjp: mapping network too wide");
  unet_mapping_vjp_kernel<<<(unsigned)rows, 256, smem, st>>>(w, sigma, aug, mcond, dcond, out);
  KDB_LAUNCH_CHECK(F_UNET_COND, st);
  return 0;
}

}  // namespace kdb
