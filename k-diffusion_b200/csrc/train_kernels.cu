// train_kernels.cu -- the reductions behind the parameter gradients of kdb_model_forward_train, fp32: the weight gradient of a Linear
// over the token rows (also with tf32 operands on the tensor cores, for the tf32 training precision), RMSNorm channel-scale gradients per image, column sums, TokenSplit's fac, and class_emb's per-class sums.
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

// tf32 weight gradient on mma.sync.m16n8k8: the same [N, K] output tiles and row chunks as wgrad_kernel, with the chunk's rows as the
// MMA's k dimension.  dY^T is the A operand (row n, column m) and X the B operand (row m, column k), so both are m-major, which wgmma
// does not take for tf32 (its tf32 operands must be K-major); mma.sync reads its fragments from registers, so the tiles are staged in
// shared memory in their global orientation, [32 rows m][64 + 8 columns], where every fragment read of a warp hits 32 distinct banks.
// Operands are truncated to tf32 as they are staged.  4 warps, each a 32 x 32 block of the 64 x 64 tile; the next 32-row slab is read
// into registers while the current one is multiplied (two shared-memory buffers).
constexpr int WT_TILE = 64, WT_SLAB = 32, WT_LD = WT_TILE + 8, WT_THREADS = 128;

__device__ __forceinline__ uint32_t tf32_trunc(float v) { return __float_as_uint(v) & 0xffffe000u; }

template <typename YL, typename XL>
__global__ void __launch_bounds__(WT_THREADS) wgrad_tf32_kernel(YL dY, XL X, float* __restrict__ part, int64_t M, int N, int K, int64_t chunk) {
  __shared__ uint32_t sy[2][WT_SLAB][WT_LD], sx[2][WT_SLAB][WT_LD];
  const int k0 = blockIdx.x * WT_TILE, n0 = blockIdx.y * WT_TILE;
  const int64_t r0 = (int64_t)blockIdx.z * chunk;
  const int rows = (int)std::min(chunk, M - r0);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int wn = (warp >> 1) * 32, wk = (warp & 1) * 32;
  const int lc = tid & 63, lr = tid >> 6;   // loader: column lc of rows lr, lr + 2, ..., lr + 30 of a slab
  uint32_t ry[WT_SLAB / 2], rx[WT_SLAB / 2];
  auto load = [&](int j0) {
#pragma unroll
    for (int i = 0; i < WT_SLAB / 2; ++i) {
      const int r = lr + 2 * i;
      const bool ok = j0 + r < rows;
      const int64_t m = r0 + j0 + r;
      ry[i] = ok && n0 + lc < N ? tf32_trunc(dY(m, n0 + lc)) : 0u;
      rx[i] = ok && k0 + lc < K ? tf32_trunc(X(m, k0 + lc)) : 0u;
    }
  };
  auto store = [&](int b) {
#pragma unroll
    for (int i = 0; i < WT_SLAB / 2; ++i) {
      sy[b][lr + 2 * i][lc] = ry[i];
      sx[b][lr + 2 * i][lc] = rx[i];
    }
  };
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  const int slabs = (rows + WT_SLAB - 1) / WT_SLAB;
  load(0);
  store(0);
  __syncthreads();
  for (int s = 0; s < slabs; ++s) {
    const int b = s & 1;
    if (s + 1 < slabs) load((s + 1) * WT_SLAB);
#pragma unroll
    for (int kk = 0; kk < WT_SLAB; kk += 8) {
      uint32_t a[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {   // A fragment: rows n = wn + 16 i + g (+ 8), columns m = kk + t4 (+ 4)
        const int nb = wn + 16 * i + g;
        a[i][0] = sy[b][kk + t4][nb];
        a[i][1] = sy[b][kk + t4][nb + 8];
        a[i][2] = sy[b][kk + t4 + 4][nb];
        a[i][3] = sy[b][kk + t4 + 4][nb + 8];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {   // B fragment: rows m = kk + t4 (+ 4), column k = wk + 8 j + g
        const uint32_t b0 = sx[b][kk + t4][wk + 8 * j + g], b1 = sx[b][kk + t4 + 4][wk + 8 * j + g];
#pragma unroll
        for (int i = 0; i < 2; ++i)
          asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                       : "+f"(acc[i][j][0]), "+f"(acc[i][j][1]), "+f"(acc[i][j][2]), "+f"(acc[i][j][3])
                       : "r"(a[i][0]), "r"(a[i][1]), "r"(a[i][2]), "r"(a[i][3]), "r"(b0), "r"(b1));
      }
    }
    if (s + 1 < slabs) store(b ^ 1);   // buffer b ^ 1 was last read in slab s - 1, before the barrier that ended it
    __syncthreads();
  }
  float* out = part + (int64_t)blockIdx.z * N * K;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // accumulator e: row g (+ 8 for e >= 2), column 2 t4 (+ 1 for odd e)
        const int n = n0 + wn + 16 * i + g + 8 * (e >> 1), k = k0 + wk + 8 * j + 2 * t4 + (e & 1);
        if (n < N && k < K) out[(int64_t)n * K + k] = acc[i][j][e];
      }
}

// Row chunks of a weight gradient: enough CTAs for two waves, at least 256 rows a chunk, partials within kTrainPartFloats
int64_t wgrad_chunk(int64_t M, int N, int K) {
  const int64_t tiles = ceil_div(N, kTileM) * ceil_div(K, kTileN);
  int64_t chunks = std::min(ceil_div(2 * kNumSMs, tiles), ceil_div(M, 256));
  chunks = std::max<int64_t>(1, std::min(chunks, kTrainPartFloats / ((int64_t)N * K)));
  return align_up((size_t)ceil_div(M, chunks), 16);
}

// tf32: the tensor-core kernel on the same chunks; the partials are summed in chunk order either way
template <bool TF32, typename YL, typename XL>
int wgrad(YL dY, XL X, float* dW, int64_t M, int N, int K, float* part, cudaStream_t st) {
  if (dW == nullptr) return 0;
  KDB_REQUIRE(M > 0 && N > 0 && K > 0, KDB_ERR_BAD_SHAPE, "wgrad: empty problem");
  const int64_t chunk = wgrad_chunk(M, N, K), chunks = ceil_div(M, chunk);
  KDB_REQUIRE(chunk <= (int64_t)1 << 30, KDB_ERR_BAD_SHAPE, "wgrad: %lld rows", (long long)M);
  dim3 grid((unsigned)ceil_div(K, kTileN), (unsigned)ceil_div(N, kTileM), (unsigned)chunks);
  float* out = chunks == 1 ? dW : part;
  if constexpr (TF32) {
    static_assert(WT_TILE == kTileM && WT_TILE == kTileN, "the tf32 kernel takes wgrad_kernel's tiles");
    wgrad_tf32_kernel<YL, XL><<<grid, WT_THREADS, 0, st>>>(dY, X, out, M, N, K, chunk);
    KDB_LAUNCH_CHECK(F_WGRAD_TF32, st);
  } else {
    wgrad_kernel<YL, XL><<<grid, 256, 0, st>>>(dY, X, out, M, N, K, chunk);
    KDB_LAUNCH_CHECK(F_GEMM_SIMT, st);
  }
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
  return wgrad<false>(Rows{dY, ldy}, Rows{X, ldx}, dW, M, N, K, part, st);
}

int launch_wgrad_merge(const float* dY, int64_t ldy, const float* fine, float* dW, int64_t M, int N, int hc, int wc, int Cf, float* part,
                       cudaStream_t st) {
  return wgrad<false>(Rows{dY, ldy}, MergeX{fine, hc, wc, Cf}, dW, M, N, 4 * Cf, part, st);
}

int launch_wgrad_tf32(const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, int64_t M, int N, int K, float* part,
                      cudaStream_t st) {
  return wgrad<true>(Rows{dY, ldy}, Rows{X, ldx}, dW, M, N, K, part, st);
}

int launch_wgrad_tf32_merge(const float* dY, int64_t ldy, const float* fine, float* dW, int64_t M, int N, int hc, int wc, int Cf, float* part,
                            cudaStream_t st) {
  return wgrad<true>(Rows{dY, ldy}, MergeX{fine, hc, wc, Cf}, dW, M, N, 4 * Cf, part, st);
}

int launch_wgrad_patch_in(const float* dtok, const float* x, float* dW, int B, int C, int H, int Wd, int ph, int pw, int N, float* part,
                          cudaStream_t st) {
  return wgrad<false>(Rows{dtok, N}, PatchX{x, C, H, Wd, ph, pw}, dW, (int64_t)B * (H / ph) * (Wd / pw), N, ph * pw * C, part, st);
}

int launch_wgrad_patch_out(const float* u, const float* tokens, const float* scale, const float* rstd, float* dW, int B, int C, int H, int Wd,
                           int ph, int pw, int C0, float* part, cudaStream_t st) {
  return wgrad<false>(PatchX{u, C, H, Wd, ph, pw}, NormX{tokens, scale, rstd, C0}, dW, (int64_t)B * (H / ph) * (Wd / pw), ph * pw * C, C0, part, st);
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
