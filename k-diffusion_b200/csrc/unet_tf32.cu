// unet_tf32.cu -- the image_v1 U-Net convolution on the tensor cores at KDB_PREC_TF32: the implicit GEMM of unet_conv_kernel
// (unet_kernels.cu) with tf32 wgmma, fp32 accumulation and fp32 activations, weights and outputs in HBM.
//
// Rounding: the weights are rounded to the nearest tf32 (ties away from zero) once, by launch_unet_round_tf32 in kdb_unet_finalize; the
// activations reach the tensor cores as TMA copied them, and the MMA ignores the low 13 mantissa bits of each, i.e. truncates them.
#include <algorithm>

#include "tc_common.cuh"
#include "unet_kernels.cuh"

namespace kdb {

namespace {

// An M tile is a box of 128 pixels, bw x bh pixels of each of bb consecutive images (bw, bh, bb powers of two), so each (tap, source,
// 32-channel block) of A is one 4-D TMA box of the token tensor [B, H, W, C] at the tap-shifted origin: the zero fill of the box's
// out-of-bounds part is the convolution's zero padding, the channels past the source's count and the pixels past the image.  B is one
// 3-D box of the tap-major weight [N, ks*ks, Ct] at (source offset + channel block, tap, n0); its channels past the source's count
// belong to the next source or are zero fill, and meet zeros in A.
constexpr int CT_BM = 128, CT_BN = 128, CT_BK = 32;                  // pixels, output channels, fp32 channels per k-block (one 128 B row)
constexpr int CT_A_BYTES = CT_BM * CT_BK * 4, CT_B_BYTES = CT_BN * CT_BK * 4;   // 16 KiB each
constexpr int CT_STAGE_BYTES = CT_A_BYTES + CT_B_BYTES;
constexpr int CT_STAGES = 6;
constexpr int CT_THREADS = 384;      // warpgroups 0, 1: MMA + epilogue of alternate tiles, warpgroup 2: TMA producer (one thread)
constexpr size_t CT_SMEM = 1024 + (size_t)CT_STAGES * CT_STAGE_BYTES + sizeof(tc::TmaRing<CT_STAGES>);

struct ConvTf32Args {
  const float* bias;
  const float* r1;
  const float* r2;
  float* out;
  int rc1, N, B, H, W;
  int c1;              // channels of source 1: the weight channel offset of source 2
  int kb1, kb2;        // 32-channel blocks per tap of source 1 / 2
  int bw, bh, bb;      // the pixel box of an M tile
  int tx, ty, tn;      // tiles along x, y and N (the batch is the slowest)
};

struct TileCoord {
  int x0, y0, b0, n0;
};
__device__ __forceinline__ TileCoord tile_coord(const ConvTf32Args& p, int t) {
  const int nt = t % p.tn, mt = t / p.tn;
  const int xt = mt % p.tx, yt = (mt / p.tx) % p.ty, bt = mt / (p.tx * p.ty);
  return TileCoord{xt * p.bw, yt * p.bh, bt * p.bb, nt * CT_BN};
}

// rows r, r + 8 of one 64-row accumulator fragment (column pair cq of every 8-column block) -> out, in the fp32 kernel's order:
// (acc + bias) + residual
__device__ __forceinline__ void store_rows(const ConvTf32Args& p, const TileCoord& tc_, int r, int cq, int box_px, const float (&acc)[64]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r + 8 * h;
    const int bi = row / box_px, rem = row - bi * box_px;
    const int yy = rem / p.bw;
    const int b = tc_.b0 + bi, y = tc_.y0 + yy, x = tc_.x0 + rem - yy * p.bw;
    if (b >= p.B || y >= p.H || x >= p.W) continue;
    const int64_t m = ((int64_t)b * p.H + y) * p.W + x;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = tc_.n0 + 8 * j + cq;
      if (n < p.N) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ne = n + e;
          if (ne >= p.N) break;
          float v = acc[4 * j + 2 * h + e];
          if (p.bias != nullptr) v += __ldg(p.bias + ne);
          if (p.r1 != nullptr) v += ne < p.rc1 ? p.r1[m * p.rc1 + ne] : p.r2[m * (p.N - p.rc1) + (ne - p.rc1)];
          p.out[m * p.N + ne] = v;
        }
      }
    }
  }
}

// The tile loop of gemm_wg_kernel (tc_kernels.cu): warp 8 streams the k-blocks of the CTA's tiles through one ring, the two MMA
// warpgroups take alternate tiles and hand the MMA issue to each other with BAR_TURN.  The epilogue adds bias and residual to the
// accumulator fragments and stores the pixels inside the image straight to global memory (a quad of threads writes 8 consecutive
// channels of a pixel).
template <int KS>
__global__ void __launch_bounds__(CT_THREADS, 1) unet_conv_tf32_kernel(const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm2,
                                                                       const __grid_constant__ CUtensorMap tmw, const ConvTf32Args p) {
  KDB_PDL_TRIGGER();
  uint8_t* base = tc::smem_1k();
  auto* ring = reinterpret_cast<tc::TmaRing<CT_STAGES>*>(base + CT_STAGES * CT_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = KS * KS * (p.kb1 + p.kb2);
  const int n_local = tc::tiles_owned(p.tx * p.ty * ((p.B + p.bb - 1) / p.bb) * p.tn);

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tm1);
    tc::tma_prefetch_desc(&tm2);
    tc::tma_prefetch_desc(&tmw);
    ring->init(tc::REL_WARPS);
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::pdl_wait();   // the activations and the residual are written by the kernels before us

  if (warp >= 8) {
    tc::setmaxnreg_dec<tc::PRODUCER_REGS>();
    if (warp == 8 && tc::elect_one()) {
      int it = 0;
      for (int i = 0; i < n_local; ++i) {
        const TileCoord tc_ = tile_coord(p, (int)blockIdx.x + i * (int)gridDim.x);
        for (int tap = 0; tap < KS * KS; ++tap) {
          const int dy = tap / KS - KS / 2, dx = tap % KS - KS / 2;
          for (int s = 0; s < 2; ++s) {
            const int nk = s ? p.kb2 : p.kb1;
            for (int cb = 0; cb < nk; ++cb, ++it) {
              const auto ps = PipeState<CT_STAGES>::at(it);
              uint64_t* bar = ring->acquire(ps, CT_STAGE_BYTES);
              uint8_t* a = base + (size_t)ps.slot * CT_STAGE_BYTES;
              tc::tma_load_4d(a, s ? &tm2 : &tm1, bar, cb * CT_BK, tc_.x0 + dx, tc_.y0 + dy, tc_.b0);
              tc::tma_load_3d(a + CT_A_BYTES, &tmw, bar, (s ? p.c1 : 0) + cb * CT_BK, tap, tc_.n0);
            }
          }
        }
      }
    }
    return;
  }
  tc::setmaxnreg_inc<tc::MMA_REGS>();

  const int wg = warp >> 2;
  const int r0 = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);   // fragment rows r0, r0 + 8 (+ 64 in acc1), column pair cq
  const int box_px = p.bw * p.bh;
  for (int i = wg; i < n_local; i += 2) {
    const TileCoord tc_ = tile_coord(p, (int)blockIdx.x + i * (int)gridDim.x);
    float acc0[64], acc1[64];
#pragma unroll
    for (int k = 0; k < 64; ++k) acc0[k] = acc1[k] = 0.f;
    if (i > 0) tc::named_barrier_sync(tc::BAR_TURN + wg, 256);   // the other warpgroup has issued the main loop of tile i - 1
    const int it0 = i * nkb;
    for (int kb = 0; kb < nkb; ++kb) {
      const auto ps = PipeState<CT_STAGES>::at(it0 + kb);
      ring->wait(ps);
      const uint32_t a_addr = tc::smem_u32(base + (size_t)ps.slot * CT_STAGE_BYTES);
      const uint64_t ad0 = tc::smem_desc_k_sw128(a_addr), ad1 = tc::smem_desc_k_sw128(a_addr + 8 * 1024);   // pixels 0-63 / 64-127
      const uint64_t bd = tc::smem_desc_k_sw128(a_addr + CT_A_BYTES);
      tc::wg_fence_acc(acc0);
      tc::wg_fence_acc(acc1);
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < CT_BK / 8; ++k) {
        tc::wgmma_128_tf32(acc0, ad0 + 2ull * k, bd + 2ull * k, 1u);
        tc::wgmma_128_tf32(acc1, ad1 + 2ull * k, bd + 2ull * k, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<1>();                  // k-block kb - 1 has completed: its stage may be refilled
      tc::wg_fence_acc(acc0);
      tc::wg_fence_acc(acc1);
      if (kb > 0 && lane == 0) ring->release(PipeState<CT_STAGES>::at(it0 + kb - 1));
    }
    if (i + 1 < n_local) tc::named_barrier_arrive(tc::BAR_TURN + (wg ^ 1), 256);
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    if (lane == 0) ring->release(PipeState<CT_STAGES>::at(it0 + nkb - 1));

    // ---------------- epilogue: out = acc + bias + residual for the tile's pixels inside the image
    store_rows(p, tc_, r0, cq, box_px, acc0);
    store_rows(p, tc_, 64 + r0, cq, box_px, acc1);
  }
}

__global__ void __launch_bounds__(256) round_tf32_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(src[i]));
    dst[i] = __uint_as_float(r);
  }
}

// ------------------------------------------------------------------------------------------------
// global self-attention (SelfAttention2d, layers.py:181-200), d_head 64, on mma.sync m16n8k8 tf32
// ------------------------------------------------------------------------------------------------
// A CTA of 4 warps takes 64 queries of one (image, head); each warp owns 16 of them.  The CTA walks the keys in blocks of 64: K and V
// of the block are staged in shared memory (rows of 68 floats: the fragment reads of both hit 32 distinct banks), S = Q K^T is a
// register fragment, the softmax keeps a running maximum per row (q and k are not normalised: no logit bound) and rescales O and l when
// it grows, and O += P V takes P straight from the S fragment.  No transpose of V is needed: the B operand of mma.sync is loaded per
// thread from registers, and the k index of the P V product is relabelled inside each 8-key group (A column t <-> key 2t, column
// t + 4 <-> key 2t + 1), so the accumulator pair a thread holds of S is exactly its A fragment of P, and V is read at the matching keys.
// q, k, v and P are truncated to tf32 (low 13 bits cleared) like the convolution's activations; l sums the truncated P.
constexpr int AT_D = 64, AT_Q = 64, AT_KB = 64, AT_LD = 68, AT_THREADS = 128;
constexpr size_t AT_SMEM = (size_t)2 * AT_KB * AT_LD * sizeof(float);

__device__ __forceinline__ uint32_t tf32_bits(float v) { return __float_as_uint(v) & 0xffffe000u; }

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(AT_THREADS) unet_attn_tf32_kernel(const float* __restrict__ qkv, float* __restrict__ out, int T, int nh) {
  extern __shared__ float at_sm[];
  float* Ks = at_sm;                       // [AT_KB][AT_LD]
  float* Vs = at_sm + AT_KB * AT_LD;
  const int head = blockIdx.y, b = blockIdx.z, C = nh * AT_D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int q0 = blockIdx.x * AT_Q + warp * 16;
  const float* base = qkv + (int64_t)b * T * 3 * C;
  // Q A fragments of the 8 k-steps along d: rows g, g + 8, columns t4, t4 + 4
  uint32_t qa[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = q0 + g + 8 * (i & 1), d = 8 * kk + t4 + 4 * (i >> 1);
      qa[kk][i] = q < T ? tf32_bits(base[(int64_t)q * 3 * C + head * AT_D + d]) : 0u;
    }
  float o[8][4], mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  constexpr float LOG2E = 1.4426950408889634f;
  for (int k0 = 0; k0 < T; k0 += AT_KB) {
    __syncthreads();                       // the previous block's K / V are no longer read
    for (int i = threadIdx.x; i < AT_KB * AT_D / 4; i += AT_THREADS) {
      const int r = i / (AT_D / 4), c4 = (i % (AT_D / 4)) * 4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + r < T) {
        const float* row = base + (int64_t)(k0 + r) * 3 * C + head * AT_D + c4;
        kv = *reinterpret_cast<const float4*>(row + C);
        vv = *reinterpret_cast<const float4*>(row + 2 * C);
      }
      *reinterpret_cast<float4*>(Ks + r * AT_LD + c4) = kv;
      *reinterpret_cast<float4*>(Vs + r * AT_LD + c4) = vv;
    }
    __syncthreads();
    // S = Q K^T for 64 keys: 8 fragments of 8 keys
    float sf[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sf[j][0] = sf[j][1] = sf[j][2] = sf[j][3] = 0.f;
      const float* kr = Ks + (8 * j + g) * AT_LD;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        mma_tf32(sf[j], qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], tf32_bits(kr[8 * kk + t4]), tf32_bits(kr[8 * kk + t4 + 4]));
    }
    // running maximum of rows g (entries 0, 1) and g + 8 (entries 2, 3)
    float n0 = mx0, n1 = mx1;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (k0 + 8 * j + 2 * t4 + e >= T) sf[j][e] = sf[j][2 + e] = -INFINITY;
        n0 = fmaxf(n0, sf[j][e]);
        n1 = fmaxf(n1, sf[j][2 + e]);
      }
    n0 = fmaxf(n0, __shfl_xor_sync(0xffffffffu, n0, 1));
    n0 = fmaxf(n0, __shfl_xor_sync(0xffffffffu, n0, 2));
    n1 = fmaxf(n1, __shfl_xor_sync(0xffffffffu, n1, 1));
    n1 = fmaxf(n1, __shfl_xor_sync(0xffffffffu, n1, 2));
    const float a0 = exp2f((mx0 - n0) * LOG2E), a1 = exp2f((mx1 - n1) * LOG2E);   // 0 on the first block (mx = -inf)
    l0 *= a0;
    l1 *= a1;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      o[n][0] *= a0;
      o[n][1] *= a0;
      o[n][2] *= a1;
      o[n][3] *= a1;
    }
    mx0 = n0;
    mx1 = n1;
    const float mb0 = n0 * LOG2E, mb1 = n1 * LOG2E;
    // P (truncated to tf32) and O += P V, one 8-key group per k-step
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t p[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        p[e] = tf32_bits(exp2f(fmaf(sf[j][e], LOG2E, -((e >> 1) ? mb1 : mb0))));
        if (e >> 1) l1 += __uint_as_float(p[e]);
        else l0 += __uint_as_float(p[e]);
      }
      const float* v0 = Vs + (8 * j + 2 * t4) * AT_LD;   // keys 8j + 2 t4 (A column t4) and + 1 (A column t4 + 4)
#pragma unroll
      for (int n = 0; n < 8; ++n) mma_tf32(o[n], p[0], p[2], p[1], p[3], tf32_bits(v0[8 * n + g]), tf32_bits(v0[AT_LD + 8 * n + g]));
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + g + 8 * h;
    if (q >= T) continue;
    float* orow = out + ((int64_t)b * T + q) * C + head * AT_D;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<float2*>(orow + 8 * n + 2 * t4) = make_float2(o[n][2 * h] * (h ? inv1 : inv0), o[n][2 * h + 1] * (h ? inv1 : inv0));
  }
}

int pow2_at_least(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// [B, H, W, C] fp32 tokens as the 4-D map (C, W, H, B) with the tile's pixel box
int tmap_tokens_f32(CUtensorMap* t, const float* base, int C, const ConvArgs& a, const ConvTf32Args& p) {
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.B};
  const uint64_t strides[3] = {(uint64_t)C * 4, (uint64_t)C * 4 * a.W, (uint64_t)C * 4 * a.W * a.H};
  const uint32_t box[4] = {CT_BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bb};
  return make_tmap_f32(t, base, 4, dims, strides, box);
}

}  // namespace

int launch_unet_conv_tf32(const ConvArgs& a, int ks, cudaStream_t st) {
  KDB_REQUIRE(ks == 1 || ks == 3, KDB_ERR_BAD_ARG, "unet_conv_tf32: kernel size %d", ks);
  KDB_REQUIRE(a.in1 && a.w && a.out && a.B > 0 && a.H > 0 && a.W > 0 && a.N > 0 && a.c1 > 0, KDB_ERR_BAD_ARG, "unet_conv_tf32: bad arguments");
  KDB_REQUIRE(a.c2 == 0 || a.in2, KDB_ERR_BAD_ARG, "unet_conv_tf32: %d channels of a second source without its pointer", a.c2);
  KDB_REQUIRE(a.c1 % 4 == 0 && a.c2 % 4 == 0 && a.rc1 % 4 == 0, KDB_ERR_BAD_SHAPE,
              "unet_conv_tf32: channel counts %d + %d must be multiples of 4", a.c1, a.c2);
  KDB_REQUIRE(!a.r1 || a.rc1 == a.N || (a.r2 && a.rc1 < a.N), KDB_ERR_BAD_ARG, "unet_conv_tf32: bad residual split");
  ConvTf32Args p{};
  p.bias = a.bias, p.r1 = a.r1, p.r2 = a.r2, p.out = a.out;
  p.rc1 = a.rc1, p.N = a.N, p.B = a.B, p.H = a.H, p.W = a.W, p.c1 = a.c1;
  p.kb1 = (int)ceil_div(a.c1, CT_BK), p.kb2 = (int)ceil_div(a.c2, CT_BK);
  p.bw = std::min(pow2_at_least(a.W), CT_BM);
  p.bh = std::min(pow2_at_least(a.H), CT_BM / p.bw);
  p.bb = CT_BM / (p.bw * p.bh);
  p.tx = (int)ceil_div(a.W, p.bw), p.ty = (int)ceil_div(a.H, p.bh), p.tn = (int)ceil_div(a.N, CT_BN);
  const int64_t tiles = (int64_t)p.tx * p.ty * ceil_div(a.B, p.bb) * p.tn;
  KDB_REQUIRE(tiles <= (1ll << 30), KDB_ERR_BAD_SHAPE, "unet_conv_tf32: %lld tiles", (long long)tiles);
  CUtensorMap t1, t2, tw;
  int rc;
  if ((rc = tmap_tokens_f32(&t1, a.in1, a.c1, a, p))) return rc;
  if ((rc = tmap_tokens_f32(&t2, a.c2 ? a.in2 : a.in1, a.c2 ? a.c2 : a.c1, a, p))) return rc;
  const int Ct = a.c1 + a.c2;
  const uint64_t wdims[3] = {(uint64_t)Ct, (uint64_t)(ks * ks), (uint64_t)a.N};
  const uint64_t wstrides[2] = {(uint64_t)Ct * 4, (uint64_t)Ct * 4 * ks * ks};
  const uint32_t wbox[3] = {CT_BK, 1, CT_BN};
  if ((rc = make_tmap_f32(&tw, a.w, 3, wdims, wstrides, wbox))) return rc;
  if (ks == 3) {
    static bool opened = false;
    if ((rc = set_smem_once(unet_conv_tf32_kernel<3>, opened, (int)CT_SMEM))) return rc;
    KDB_CUDA(launch_pdl(unet_conv_tf32_kernel<3>, persistent_grid(tiles), dim3(CT_THREADS), CT_SMEM, st, t1, t2, tw, p));
  } else {
    static bool opened = false;
    if ((rc = set_smem_once(unet_conv_tf32_kernel<1>, opened, (int)CT_SMEM))) return rc;
    KDB_CUDA(launch_pdl(unet_conv_tf32_kernel<1>, persistent_grid(tiles), dim3(CT_THREADS), CT_SMEM, st, t1, t2, tw, p));
  }
  KDB_LAUNCH_CHECK(F_UNET_CONV_TF32, st);
  return 0;
}

bool unet_attn_tf32_supported(int d_head) { return d_head == AT_D; }

int launch_unet_attn_tf32(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st) {
  KDB_REQUIRE(qkv && out && B > 0 && T > 0 && nh > 0, KDB_ERR_BAD_ARG, "unet_attn_tf32: bad arguments");
  KDB_REQUIRE(unet_attn_tf32_supported(d_head), KDB_ERR_UNSUPPORTED, "unet_attn_tf32: d_head %d (the kernel is built for 64)", d_head);
  KDB_REQUIRE(B <= 65535 && nh <= 65535, KDB_ERR_BAD_SHAPE, "unet_attn_tf32: %d images x %d heads exceed the grid", B, nh);
  unet_attn_tf32_kernel<<<dim3((unsigned)ceil_div(T, AT_Q), (unsigned)nh, (unsigned)B), AT_THREADS, AT_SMEM, st>>>(qkv, out, T, nh);
  KDB_LAUNCH_CHECK(F_UNET_ATTN_TF32, st);
  return 0;
}

int launch_unet_round_tf32(const float* src, float* dst, int64_t n, cudaStream_t st) {
  round_tf32_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), (int64_t)kNumSMs * 32), 256, 0, st>>>(src, dst, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

}  // namespace kdb
