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

}  // namespace kdb
