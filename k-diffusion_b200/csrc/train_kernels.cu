// train_kernels.cu -- the reductions behind the parameter gradients of kdb_model_forward_train, fp32: the weight gradient of a Linear
// over the token rows, RMSNorm channel-scale gradients per image, column sums, TokenSplit's fac, and class_emb's per-class sums.
// No atomics.  A sum over many rows is split into chunks fixed by the shapes alone, each chunk summed in row order, then the chunk
// partials summed in chunk order by segsum_kernel, so two calls on the same inputs give the same bits.
#include <algorithm>

#include "model_kernels.cuh"
#include "simt_tile.cuh"

namespace kdb {

namespace {

constexpr float kEps = 1e-6f;      // RMSNorm eps (image_transformer_v2.py:143)
constexpr int kNormChunk = 64;     // rows per partial of launch_norm_scale_grad
constexpr int kSumChunk = 256;     // rows per partial of launch_colsum

unsigned stride_blocks(int64_t n) { return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(n, 256), 1), kNumSMs * 16); }

// out[s * ldo + c] = sum over the rows r of segment s of P[r * C + c], r ascending; segment s holds rows [s R, min((s + 1) R, rows))
__global__ void __launch_bounds__(256) segsum_kernel(const float* __restrict__ P, float* __restrict__ out, int64_t ldo, int64_t rows, int64_t R,
                                                     int64_t C, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t s = i / C, c = i - s * C;
    const int64_t r1 = std::min(rows, (s + 1) * R);
    float acc = 0.f;
    for (int64_t r = s * R; r < r1; ++r) acc += P[r * C + c];
    out[s * ldo + c] = acc;
  }
}

int segsum(const float* P, float* out, int64_t ldo, int64_t rows, int64_t R, int64_t C, cudaStream_t st) {
  const int64_t total = ceil_div(rows, R) * C;
  segsum_kernel<<<stride_blocks(total), 256, 0, st>>>(P, out, ldo, rows, R, C, total);
  KDB_LAUNCH_CHECK(F_GEMM_SIMT, st);
  return 0;
}

// Operands of the weight-gradient GEMM: element (m, k) of the [M, K] input of the forward's Linear, or of its output gradient
struct Rows {
  const float* p;
  int64_t ld;
  __device__ float operator()(int64_t m, int k) const { return p[m * ld + k]; }
};
struct MergeX {   // the TokenMerge gather of fine tokens [B, 2hc, 2wc, Cf], in place
  const float* p;
  int hc, wc, Cf;
  __device__ float operator()(int64_t m, int k) const { return p[merge_source(m * 4 * Cf + k, hc, wc, Cf)]; }
};
struct PatchX {   // the patch rows [B T, (nh nw c)] of an NCHW image [B, C, H, W], in place
  const float* p;
  int C, H, W, ph, pw;
  __device__ float operator()(int64_t m, int k) const {
    int b, ty, tx;
    token_coords(m, H / ph, W / pw, b, ty, tx);
    return p[patch_pixel(b, ty, tx, k, C, H, W, ph, pw)];
  }
};
struct NormX {    // RMSNorm's output x * (scale * rstd) of rows x [M, K], rstd per row as the forward computed it
  const float *x, *scale, *rstd;
  int K;
  __device__ float operator()(int64_t m, int k) const { return x[m * K + k] * (__ldg(scale + k) * rstd[m]); }
};

// Chunk z of the rows: part[z, n, k] = sum over m in the chunk of dY[m, n] X(m, k), on the tile loop of simt_tile.cuh with (n, k) as
// the output tile and the chunk's rows as the reduction.
template <typename YL, typename XL>
__global__ void __launch_bounds__(256) wgrad_kernel(YL dY, XL X, float* __restrict__ part, int64_t M, int N, int K, int64_t chunk) {
  const int k0 = blockIdx.x * kTileN;
  const int n0 = blockIdx.y * kTileM;
  const int64_t r0 = (int64_t)blockIdx.z * chunk;
  const int rows = (int)std::min(chunk, M - r0);
  const int tid = threadIdx.x;
  const int rr = tid >> 4, c4 = (tid & 15) * 4;   // loader: reduction row 0..15, columns c4..c4+3
  auto fill = [&](int j0, TileSmem& As, TileSmem& Ws) {
    const bool ok = j0 + rr < rows;
    const int64_t m = r0 + j0 + rr;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[rr][c4 + i] = ok && n0 + c4 + i < N ? dY(m, n0 + c4 + i) : 0.f;
      Ws[rr][c4 + i] = ok && k0 + c4 + i < K ? X(m, k0 + c4 + i) : 0.f;
    }
  };
  float* out = part + (int64_t)blockIdx.z * N * K;
  simt_tile(n0, k0, N, K, rows, fill, [&](int64_t n, int k, float acc) { out[n * K + k] = acc; });
}

// Row chunks of a weight gradient: enough CTAs for two waves, at least 256 rows a chunk, partials within kTrainPartFloats
template <typename YL, typename XL>
int wgrad(YL dY, XL X, float* dW, int64_t M, int N, int K, float* part, cudaStream_t st) {
  if (dW == nullptr) return 0;
  KDB_REQUIRE(M > 0 && N > 0 && K > 0, KDB_ERR_BAD_SHAPE, "wgrad: empty problem");
  const int64_t tiles = ceil_div(N, kTileM) * ceil_div(K, kTileN);
  int64_t chunks = std::min(ceil_div(2 * kNumSMs, tiles), ceil_div(M, 256));
  chunks = std::max<int64_t>(1, std::min(chunks, kTrainPartFloats / ((int64_t)N * K)));
  const int64_t chunk = align_up((size_t)ceil_div(M, chunks), 16);
  chunks = ceil_div(M, chunk);
  KDB_REQUIRE(chunk <= (int64_t)1 << 30, KDB_ERR_BAD_SHAPE, "wgrad: %lld rows", (long long)M);
  dim3 grid((unsigned)ceil_div(K, kTileN), (unsigned)ceil_div(N, kTileM), (unsigned)chunks);
  wgrad_kernel<YL, XL><<<grid, 256, 0, st>>>(dY, X, chunks == 1 ? dW : part, M, N, K, chunk);
  KDB_LAUNCH_CHECK(F_GEMM_SIMT, st);
  return chunks == 1 ? 0 : segsum(part, dW, 0, chunks, chunks, (int64_t)N * K, st);
}

// Chunk ch (of image ch / cpb): part[ch, c] = sum over its rows of dy[r, c] (x[r, c] rstd_r), rstd_r as rmsnorm_kernel computes it
__global__ void __launch_bounds__(256) norm_scale_part_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dy, int64_t ldy,
                                                              float* __restrict__ part, int64_t rows_per_batch, int cpb, int C) {
  __shared__ float rs[kNormChunk];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t b = blockIdx.x / cpb, j = blockIdx.x - b * cpb;
  const int64_t r0 = b * rows_per_batch + j * kNormChunk;
  const int n = (int)std::min<int64_t>(kNormChunk, rows_per_batch - j * kNormChunk);
  for (int i = warp; i < n; i += 8) {
    const float* xr = x + (r0 + i) * ldx;
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) ss = fmaf(xr[c], xr[c], ss);
    ss = warp_sum(ss);
    if (lane == 0) rs[i] = rsqrtf(ss / (float)C + kEps);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float acc = 0.f;
    for (int i = 0; i < n; ++i) acc = fmaf(dy[(r0 + i) * ldy + c], x[(r0 + i) * ldx + c] * rs[i], acc);
    part[(int64_t)blockIdx.x * C + c] = acc;
  }
}

__global__ void __launch_bounds__(256) split_fac_part_kernel(const float* __restrict__ y, const float* __restrict__ skip,
                                                             const float* __restrict__ dup, float* __restrict__ part, int H, int Wd, int C,
                                                             int64_t total) {
  __shared__ float red[8];
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t src = merge_source(i, H / 2, Wd / 2, C);
    acc = fmaf(y[i] - skip[src], dup[src], acc);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(256) class_emb_grad_kernel(const float* __restrict__ demb, int64_t ldd, const int64_t* __restrict__ cls,
                                                             float* __restrict__ out, int rows, int mw, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t k = i / mw;
    const int j = (int)(i - k * mw);
    float acc = 0.f;
    for (int r = 0; r < rows; ++r)
      if (cls[r] == k) acc += demb[(int64_t)r * ldd + j];
    out[i] = acc;
  }
}

}  // namespace

int launch_wgrad(const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, int64_t M, int N, int K, float* part, cudaStream_t st) {
  return wgrad(Rows{dY, ldy}, Rows{X, ldx}, dW, M, N, K, part, st);
}

int launch_wgrad_merge(const float* dY, const float* fine, float* dW, int64_t M, int N, int hc, int wc, int Cf, float* part, cudaStream_t st) {
  return wgrad(Rows{dY, N}, MergeX{fine, hc, wc, Cf}, dW, M, N, 4 * Cf, part, st);
}

int launch_wgrad_patch_in(const float* dtok, const float* x, float* dW, int B, int C, int H, int Wd, int ph, int pw, int N, float* part,
                          cudaStream_t st) {
  return wgrad(Rows{dtok, N}, PatchX{x, C, H, Wd, ph, pw}, dW, (int64_t)B * (H / ph) * (Wd / pw), N, ph * pw * C, part, st);
}

int launch_wgrad_patch_out(const float* u, const float* tokens, const float* scale, const float* rstd, float* dW, int B, int C, int H, int Wd,
                           int ph, int pw, int C0, float* part, cudaStream_t st) {
  return wgrad(PatchX{u, C, H, Wd, ph, pw}, NormX{tokens, scale, rstd, C0}, dW, (int64_t)B * (H / ph) * (Wd / pw), ph * pw * C, C0, part, st);
}

int launch_norm_scale_grad(const float* x, int64_t ldx, const float* dy, int64_t ldy, float* out, int64_t ldo, int64_t rows_per_batch,
                           int64_t rows, int C, float* part, cudaStream_t st) {
  if (out == nullptr) return 0;
  KDB_REQUIRE(rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0, KDB_ERR_BAD_SHAPE, "norm_scale_grad: bad rows");
  const int64_t B = rows / rows_per_batch, cpb = ceil_div(rows_per_batch, kNormChunk);
  KDB_REQUIRE(B * cpb * C <= kTrainPartFloats, KDB_ERR_BAD_SHAPE, "norm_scale_grad: %lld rows of %d channels", (long long)rows, C);
  norm_scale_part_kernel<<<(unsigned)(B * cpb), 256, 0, st>>>(x, ldx, dy, ldy, part, rows_per_batch, (int)cpb, C);
  KDB_LAUNCH_CHECK(F_RMSNORM, st);
  return segsum(part, out, ldo, B * cpb, cpb, C, st);
}

int launch_colsum(const float* P, int64_t rows, int C, float* out, float* part, cudaStream_t st) {
  if (out == nullptr) return 0;
  const int64_t chunks = ceil_div(rows, kSumChunk);
  KDB_REQUIRE(chunks * C <= kTrainPartFloats, KDB_ERR_BAD_SHAPE, "colsum: %lld rows of %d columns", (long long)rows, C);
  int rc = segsum(P, part, C, rows, kSumChunk, C, st);
  return rc ? rc : segsum(part, out, 0, chunks, chunks, C, st);
}

int launch_split_fac_grad(const float* y, const float* skip, const float* dup, float* out, int B, int H, int Wd, int C, float* part,
                          cudaStream_t st) {
  if (out == nullptr) return 0;
  const int64_t total = (int64_t)B * H * Wd * C;
  const unsigned blocks = stride_blocks(total);
  split_fac_part_kernel<<<blocks, 256, 0, st>>>(y, skip, dup, part, H, Wd, C, total);
  KDB_LAUNCH_CHECK(F_MERGE_GATHER, st);
  return segsum(part, out, 0, blocks, blocks, 1, st);
}

int launch_class_emb_grad(const float* demb, int64_t ldd, const int64_t* cls, float* out, int rows, int n_classes, int mw, cudaStream_t st) {
  if (out == nullptr) return 0;
  const int64_t total = (int64_t)n_classes * mw;
  class_emb_grad_kernel<<<stride_blocks(total), 256, 0, st>>>(demb, ldd, cls, out, rows, mw, total);
  KDB_LAUNCH_CHECK(F_COND, st);
  return 0;
}

}  // namespace kdb
