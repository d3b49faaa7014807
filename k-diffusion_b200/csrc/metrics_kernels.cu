// metrics_kernels.cu -- the fp32 products behind KID and FID (reference evaluation.py:93-161, which runs them with TF32 off, i.e. as
// fp32 FFMA): the polynomial-kernel MMD sums, the polynomial-kernel matrix and the feature mean and covariance, all on the SIMT tile
// loop (simt_tile.cuh).  No atomics: every sum runs in a fixed order, so two calls on the same inputs return the same bits.
#include <algorithm>
#include <climits>
#include <vector>

#include "simt_tile.cuh"

namespace kdb {

namespace {

// k(a, b) = (a . b / d + 1)^3 in fp32, in the reference's operation order (evaluation.py:93-96)
__device__ __forceinline__ float poly3(float dot, float d) {
  const float t = dot / d + 1.f;
  return t * t * t;
}

// Stores the k-block [k0, k0 + 16) of `rows` rows (at most 64 are read) starting at p into S[k][row], zeros past rows or d.  V4: d is a
// multiple of 4 and p 16-byte aligned, so every thread moves one float4.
template <bool V4>
__device__ __forceinline__ void load_rows(TileSmem& S, const float* __restrict__ p, int64_t rows, int d, int k0) {
  const int tid = threadIdx.x, lr = tid >> 2, lk = (tid & 3) * 4, k = k0 + lk;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (lr < rows) {
    const float* src = p + (int64_t)lr * d + k;
    if (V4) {
      if (k < d) {
        const float4 f = __ldg(reinterpret_cast<const float4*>(src));
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (k + q < d) v[q] = __ldg(src + q);
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) S[lk + q][lr] = v[q];
}

__device__ __forceinline__ int tiles_of(int64_t rows) { return (int)((rows + kTileM - 1) / kTileM); }
__device__ __forceinline__ int tri(int t) { return t * (t + 1) / 2; }

// sum of v over the 256 threads of a CTA, in the same order on every call; red: 8 doubles of shared scratch.  Valid on thread 0.
__device__ __forceinline__ double block_sum_d(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

// Segment s of an MMD call: rows [xoff[s], xoff[s+1]) of x against rows [yoff[s], yoff[s+1]) of y.  Its tile slots, in order: the
// upper-triangle 64x64 tiles of k(x, x) row by row, then those of k(y, y), then every tile of k(x, y); slots past them hold 0.
struct MmdArgs {
  const float* x;
  const float* y;
  const int64_t* xoff;    // [S + 1], in the workspace
  const int64_t* yoff;    // [S + 1]
  double* partial;        // [S][slots]
  int d, slots;
};

struct SegTiles {
  int64_t x0, mx, y0, ny;
  int tx, ty, nxx, nyy, nxy;
};

__device__ __forceinline__ SegTiles seg_tiles(const int64_t* xoff, const int64_t* yoff, int s) {
  SegTiles g;
  g.x0 = xoff[s]; g.mx = xoff[s + 1] - g.x0;
  g.y0 = yoff[s]; g.ny = yoff[s + 1] - g.y0;
  g.tx = tiles_of(g.mx); g.ty = tiles_of(g.ny);
  g.nxx = tri(g.tx); g.nyy = tri(g.ty); g.nxy = g.tx * g.ty;
  return g;
}

// One CTA per (tile slot, segment): the fp64 sum of the tile's kernel values -- strictly above the diagonal, and counted twice, for
// k(x, x) and k(y, y) -- into partial[s][slot].  The diagonal is never added.
template <bool V4>
__global__ void __launch_bounds__(256) mmd_tiles_kernel(const MmdArgs a) {
  __shared__ double red[8];
  const int s = blockIdx.y;
  int t = blockIdx.x;
  const SegTiles g = seg_tiles(a.xoff, a.yoff, s);
  double* out = a.partial + (int64_t)s * a.slots + blockIdx.x;
  const float *A, *B;
  int64_t M, N;
  int T = 0, bi, bj;
  bool sym = true;
  if (t < g.nxx) {
    A = B = a.x + g.x0 * a.d; M = N = g.mx; T = g.tx;
  } else if ((t -= g.nxx) < g.nyy) {
    A = B = a.y + g.y0 * a.d; M = N = g.ny; T = g.ty;
  } else if ((t -= g.nyy) < g.nxy) {
    A = a.x + g.x0 * a.d; B = a.y + g.y0 * a.d; M = g.mx; N = g.ny; T = 0; sym = false;
  } else {
    if (threadIdx.x == 0) *out = 0.0;
    return;
  }
  if (sym) {   // upper-triangle slot t -> (bi, bj), bi <= bj: row bi holds T - bi tiles
    bi = 0;
    while (t >= T - bi) t -= T - bi++;
    bj = bi + t;
  } else {
    bi = t / g.ty;
    bj = t - bi * g.ty;
  }
  const bool diag = sym && bi == bj;
  const int64_t m0 = (int64_t)bi * kTileM;
  const int n0 = bj * kTileN;
  const float fd = (float)a.d;
  double sum = 0.0;
  simt_tile(
      m0, n0, M, (int)N, a.d,
      [&](int k0, TileSmem& As, TileSmem& Ws) {
        load_rows<V4>(As, A + m0 * a.d, M - m0, a.d, k0);
        load_rows<V4>(Ws, B + (int64_t)n0 * a.d, N - n0, a.d, k0);
      },
      [&](int64_t m, int n, float dot) {
        if (!diag || n > m) sum += (double)poly3(dot, fd);
      });
  sum = block_sum_d(sum, red);
  if (threadIdx.x == 0) *out = sym ? 2.0 * sum : sum;
}

// One CTA per segment: the three sums of its tile slots in slot order, then term_1 + term_2 - term_3 in fp64 (evaluation.py:99-111).
// out[s] = (kxx off-diagonal sum, kyy off-diagonal sum, kxy sum, squared MMD).
__global__ void __launch_bounds__(256) mmd_reduce_kernel(const MmdArgs a, double* __restrict__ out) {
  __shared__ double red[8];
  const int s = blockIdx.x;
  const SegTiles g = seg_tiles(a.xoff, a.yoff, s);
  const double* p = a.partial + (int64_t)s * a.slots;
  const int bounds[4] = {0, g.nxx, g.nxx + g.nyy, g.nxx + g.nyy + g.nxy};
  double sums[3];
  for (int q = 0; q < 3; ++q) {
    double v = 0.0;
    for (int i = bounds[q] + threadIdx.x; i < bounds[q + 1]; i += blockDim.x) v += p[i];
    sums[q] = block_sum_d(v, red);
  }
  if (threadIdx.x == 0) {
    const double m = (double)g.mx, n = (double)g.ny;
    const double t1 = sums[0] / m / (m - 1.0), t2 = sums[1] / n / (n - 1.0), t3 = sums[2] * 2.0 / m / n;
    out[4 * s + 0] = sums[0];
    out[4 * s + 1] = sums[1];
    out[4 * s + 2] = sums[2];
    out[4 * s + 3] = t1 + t2 - t3;
  }
}

// out[b] = k(x[b], y[b]) [m, n] fp32; one CTA per 64x64 output tile, blockIdx.z = b
template <bool V4>
__global__ void __launch_bounds__(256) poly_kernel_kernel(const float* __restrict__ x, const float* __restrict__ y, float* __restrict__ out, int m,
                                                          int n, int d) {
  const int b = blockIdx.z;
  const float* xb = x + (int64_t)b * m * d;
  const float* yb = y + (int64_t)b * n * d;
  float* ob = out + (int64_t)b * m * n;
  const int64_t m0 = (int64_t)blockIdx.y * kTileM;
  const int n0 = blockIdx.x * kTileN;
  const float fd = (float)d;
  simt_tile(
      m0, n0, m, n, d,
      [&](int k0, TileSmem& As, TileSmem& Ws) {
        load_rows<V4>(As, xb + m0 * d, m - m0, d, k0);
        load_rows<V4>(Ws, yb + (int64_t)n0 * d, n - n0, d, k0);
      },
      [&](int64_t i, int j, float dot) { ob[i * n + j] = poly3(dot, fd); });
}

// mean[c] = (sum_r x[r, c]) / n: 32 columns per CTA, 8 row lanes each, fp64 sums added lane by lane in a fixed order
__global__ void __launch_bounds__(256) col_mean_kernel(const float* __restrict__ x, int64_t n, int d, float* __restrict__ mean) {
  __shared__ double red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  double s = 0.0;
  if (c < d)
    for (int64_t r = ty; r < n; r += 8) s += (double)__ldg(x + r * d + c);
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < d) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w][tx];
    mean[c] = (float)(t / (double)n);
  }
}

// The upper-triangle 64x64 tiles of (x - mean)^T (x - mean) / (n - 1) (torch.cov of x.T, evaluation.py:154-155), each written to both
// (i, j) and (j, i).  The reduction runs over the n samples; fill stores x - mean (fp32) of 16 samples x 64 features, zeros past n or d.
// V4: d is a multiple of 4 and x and mean are 16-byte aligned.
template <bool V4>
__global__ void __launch_bounds__(256) cov_kernel(const float* __restrict__ x, const float* __restrict__ mean, int n, int d,
                                                  float* __restrict__ cov) {
  const int T = tiles_of(d);
  int t = blockIdx.x, bi = 0;
  while (t >= T - bi) t -= T - bi++;
  const int bj = bi + t;
  const int i0 = bi * kTileM, j0 = bj * kTileN;
  const int kk = threadIdx.x >> 4, f = (threadIdx.x & 15) * 4;
  auto load = [&](TileSmem& S, const float* row, int c0, bool in) {
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (in) {
      if (V4) {
        if (c0 + f < d) {
          const float4 g = __ldg(reinterpret_cast<const float4*>(row + c0 + f));
          const float4 mu = __ldg(reinterpret_cast<const float4*>(mean + c0 + f));
          v[0] = g.x - mu.x; v[1] = g.y - mu.y; v[2] = g.z - mu.z; v[3] = g.w - mu.w;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (c0 + f + q < d) v[q] = __ldg(row + c0 + f + q) - __ldg(mean + c0 + f + q);
      }
    }
    *reinterpret_cast<float4*>(&S[kk][f]) = make_float4(v[0], v[1], v[2], v[3]);
  };
  const float denom = (float)(n - 1);
  simt_tile(
      i0, j0, d, d, n,
      [&](int k0, TileSmem& As, TileSmem& Ws) {
        const bool in = k0 + kk < n;
        const float* row = x + (int64_t)(k0 + kk) * d;
        load(As, row, i0, in);
        load(Ws, row, j0, in);
      },
      [&](int64_t i, int j, float acc) {
        if (bi == bj && j < i) return;
        const float v = acc / denom;
        cov[i * d + j] = v;
        cov[(int64_t)j * d + i] = v;
      });
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Validates a segment list and returns its tile slots per segment (the most any segment needs, at least 1) or a KDB_ERR_*.
int64_t mmd_slots(const int64_t* xo, const int64_t* yo, int S, int64_t m, int64_t n) {
  KDB_REQUIRE(xo && yo, KDB_ERR_BAD_ARG, "mmd: NULL segment offsets");
  KDB_REQUIRE(S >= 1 && S <= 65535, KDB_ERR_BAD_ARG, "mmd: %d segments (1..65535)", S);
  int64_t slots = 1;
  for (int s = 0; s < S; ++s) {
    const int64_t mx = xo[s + 1] - xo[s], ny = yo[s + 1] - yo[s];
    KDB_REQUIRE(xo[s] >= 0 && yo[s] >= 0 && mx >= 0 && ny >= 0 && xo[s + 1] <= m && yo[s + 1] <= n, KDB_ERR_BAD_SHAPE,
                "mmd: segment %d rows [%lld, %lld) of x / [%lld, %lld) of y are not ordered row ranges of %lld / %lld rows", s,
                (long long)xo[s], (long long)xo[s + 1], (long long)yo[s], (long long)yo[s + 1], (long long)m, (long long)n);
    const int64_t tx = ceil_div(mx, kTileM), ty = ceil_div(ny, kTileM);
    slots = std::max(slots, tx * (tx + 1) / 2 + ty * (ty + 1) / 2 + tx * ty);
  }
  KDB_REQUIRE(slots <= INT_MAX, KDB_ERR_BAD_SHAPE, "mmd: %lld tiles per segment exceed the grid", (long long)slots);
  return slots;
}

size_t mmd_offsets_bytes(int S) { return align_up(2 * (size_t)(S + 1) * sizeof(int64_t), 256); }

}  // namespace

}  // namespace kdb

using namespace kdb;

extern "C" {

int64_t kdb_mmd_workspace_bytes(const int64_t* x_offsets_host, const int64_t* y_offsets_host, int n_segments) {
  const int64_t slots = mmd_slots(x_offsets_host, y_offsets_host, n_segments, INT64_MAX, INT64_MAX);
  if (slots < 0) return slots;
  return (int64_t)(mmd_offsets_bytes(n_segments) + (size_t)n_segments * slots * sizeof(double));
}

int kdb_mmd_sums(const float* x, int64_t m, const float* y, int64_t n, int d, const int64_t* x_offsets_host, const int64_t* y_offsets_host,
                 int n_segments, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(x && y && out && workspace, KDB_ERR_BAD_ARG, "mmd_sums: NULL x, y, out or workspace");
  KDB_REQUIRE(d >= 1 && m >= 0 && n >= 0, KDB_ERR_BAD_SHAPE, "mmd_sums: %lld x %d and %lld x %d features", (long long)m, d, (long long)n, d);
  const int64_t slots = mmd_slots(x_offsets_host, y_offsets_host, n_segments, m, n);
  if (slots < 0) return (int)slots;
  const int S = n_segments;
  const size_t need = mmd_offsets_bytes(S) + (size_t)S * slots * sizeof(double);
  KDB_REQUIRE(workspace_bytes >= need, KDB_ERR_WORKSPACE, "mmd_sums: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<int64_t> offs(2 * (size_t)(S + 1));
  std::copy(x_offsets_host, x_offsets_host + S + 1, offs.begin());
  std::copy(y_offsets_host, y_offsets_host + S + 1, offs.begin() + S + 1);
  int64_t* dev_offs = static_cast<int64_t*>(workspace);
  // from pageable memory: the call returns once `offs` has been staged, so it may be freed right after
  KDB_CUDA(cudaMemcpyAsync(dev_offs, offs.data(), offs.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  MmdArgs a;
  a.x = x; a.y = y; a.xoff = dev_offs; a.yoff = dev_offs + S + 1;
  a.partial = reinterpret_cast<double*>(static_cast<char*>(workspace) + mmd_offsets_bytes(S));
  a.d = d; a.slots = (int)slots;
  const dim3 grid((unsigned)slots, (unsigned)S);
  if (d % 4 == 0 && aligned16(x) && aligned16(y))
    mmd_tiles_kernel<true><<<grid, 256, 0, st>>>(a);
  else
    mmd_tiles_kernel<false><<<grid, 256, 0, st>>>(a);
  KDB_LAUNCH_CHECK(F_MMD_TILES, st);
  mmd_reduce_kernel<<<S, 256, 0, st>>>(a, out);
  KDB_LAUNCH_CHECK(F_MMD_REDUCE, st);
  return 0;
}

int kdb_polynomial_kernel(const float* x, const float* y, float* out, int batch, int m, int n, int d, void* stream) {
  KDB_REQUIRE(x && y && out, KDB_ERR_BAD_ARG, "polynomial_kernel: NULL x, y or out");
  KDB_REQUIRE(batch >= 1 && m >= 1 && n >= 1 && d >= 1, KDB_ERR_BAD_SHAPE, "polynomial_kernel: batch %d of %d x %d and %d x %d features", batch,
              m, d, n, d);
  KDB_REQUIRE(batch <= 65535 && ceil_div(m, kTileM) <= 65535, KDB_ERR_BAD_SHAPE, "polynomial_kernel: batch %d or %d rows exceed the grid", batch,
              m);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)ceil_div(n, kTileN), (unsigned)ceil_div(m, kTileM), (unsigned)batch);
  if (d % 4 == 0 && aligned16(x) && aligned16(y))
    poly_kernel_kernel<true><<<grid, 256, 0, st>>>(x, y, out, m, n, d);
  else
    poly_kernel_kernel<false><<<grid, 256, 0, st>>>(x, y, out, m, n, d);
  KDB_LAUNCH_CHECK(F_POLY_KERNEL, st);
  return 0;
}

int kdb_feature_mean_cov(const float* x, int64_t n, int d, float* mean, float* cov, void* stream) {
  KDB_REQUIRE(x && mean && cov, KDB_ERR_BAD_ARG, "feature_mean_cov: NULL x, mean or cov");
  KDB_REQUIRE(n >= 1 && n <= INT_MAX && d >= 1, KDB_ERR_BAD_SHAPE, "feature_mean_cov: %lld x %d features", (long long)n, d);
  cudaStream_t st = (cudaStream_t)stream;
  col_mean_kernel<<<(unsigned)ceil_div(d, 32), 256, 0, st>>>(x, n, d, mean);
  KDB_LAUNCH_CHECK(F_COL_MEAN, st);
  const int64_t T = ceil_div(d, kTileM);
  if (d % 4 == 0 && aligned16(x) && aligned16(mean))
    cov_kernel<true><<<(unsigned)(T * (T + 1) / 2), 256, 0, st>>>(x, mean, (int)n, d, cov);
  else
    cov_kernel<false><<<(unsigned)(T * (T + 1) / 2), 256, 0, st>>>(x, mean, (int)n, d, cov);
  KDB_LAUNCH_CHECK(F_COV, st);
  return 0;
}

}  // extern "C"
