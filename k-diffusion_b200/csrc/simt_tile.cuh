// simt_tile.cuh -- the tile loop of the SIMT GEMMs (gemm_simt_kernel, gemm_vjp_kernel in model_kernels.cu; unet_conv_kernel in
// unet_kernels.cu): 64x64x16 tiles, 256 threads, 4x4 micro-tile per thread, fp32 accumulate.
#pragma once
#include "common.cuh"

namespace kdb {

constexpr int kTileM = 64, kTileN = 64, kTileK = 16, kTilePad = 4;
using TileSmem = float[kTileK][kTileM + kTilePad];   // one k-block of 64 rows, k-major (kTileM == kTileN)

// The output tile whose first row is m0 and first column n0 of an M x N product with reduction length K.  fill(k0, As, Ws) stores
// the k-block [k0, k0 + 16) of the tile's 64 A rows in As[k][row] and of its 64 W rows in Ws[k][col], zeros past M, N or K.  Each
// thread accumulates its 4x4 outputs over the k-blocks in order, one fmaf per k, then emit(m, n, acc) receives every one of them
// that lies inside M x N.
template <typename Fill, typename Emit>
__device__ __forceinline__ void simt_tile(int64_t m0, int n0, int64_t M, int N, int K, Fill&& fill, Emit&& emit) {
  __shared__ __align__(16) TileSmem As, Ws;
  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += kTileK) {
    fill(k0, As, Ws);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kTileK; ++kk) {
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

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      emit(m, n, acc[i][j]);
    }
  }
}

}  // namespace kdb
