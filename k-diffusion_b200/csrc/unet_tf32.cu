// unet_tf32.cu -- the image_v1 U-Net convolution and d_head-64 self-attention on the tensor cores, at KDB_PREC_TF32 and KDB_PREC_FP16:
// the implicit GEMM of unet_conv_kernel (unet_kernels.cu) with fp32 accumulation and fp32 activations and outputs in HBM.  One kernel of
// each, whose operand format (Tf32Ops, F16Ops) is a template parameter.
//
// Rounding at tf32: the weights are rounded to the nearest tf32 (ties away from zero) once, by launch_unet_round_tf32 in
// kdb_unet_finalize; the activations reach the tensor cores as TMA copied them, and the MMA ignores the low 13 mantissa bits of each,
// i.e. truncates them.  At fp16: the weights are rounded to the nearest fp16 (ties to even) once, by launch_unet_round_f16; the MMA
// warpgroups round each staged fp32 activation to the nearest fp16 (ties to even, cvt.rn.f16x2.f32) in registers.  Both roundings
// overflow to infinity (no .satfinite): an operand of magnitude >= 65520 becomes +-inf, so it reaches the output as inf or NaN.
#include <algorithm>
#include <type_traits>

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
constexpr int CT_A_BYTES = CT_BM * CT_BK * 4;                        // 16 KiB
constexpr int CT_THREADS = 384;      // warpgroups 0, 1: MMA + epilogue of alternate tiles, warpgroup 2: TMA producer (one thread)

// The operand formats.  Tf32Ops: B is the tf32-rounded fp32 weight (a 32-channel row is 128 B, SWIZZLE_128B) and wgmma reads A from the
// staged fp32 tile.  F16Ops: B is the fp16 weight copy (a 32-channel row is 64 B, SWIZZLE_64B) and wgmma takes A from registers, converted
// from the staged fp32 tile; its smaller stages make room for two more.
struct Tf32Ops {
  static constexpr int B_ELEM = 4, STAGES = 6;
};
struct F16Ops {
  static constexpr int B_ELEM = 2, STAGES = 8;
};
template <class Op>
struct ConvTc {
  static constexpr int B_BYTES = CT_BN * CT_BK * Op::B_ELEM;
  static constexpr int STAGE_BYTES = CT_A_BYTES + B_BYTES;
  static constexpr size_t SMEM = 1024 + (size_t)Op::STAGES * STAGE_BYTES + sizeof(tc::TmaRing<Op::STAGES>);
};

struct ConvTcArgs {
  const float* bias;
  const float* r1;
  const float* r2;
  float* out;
  int rc1, N, B, H, W;
  int c1;              // channels of source 1: the weight channel offset of source 2
  int kb1, kb2;        // 32-channel blocks per tap of source 1 / 2
  int bw, bh, bb;      // the pixel box of an M tile
  int tx, ty, tn;      // tiles along x, y and N (the batch is the slowest)
  int shift2;          // F16Ops: c1 % 8.  Source 2's boxes start this many channels early, its weight boxes at a 16-byte aligned channel
                       // (TMA needs that of a swizzled box); the early channels of its activation box are zero fill
};

struct TileCoord {
  int x0, y0, b0, n0;
};
__device__ __forceinline__ TileCoord tile_coord(const ConvTcArgs& p, int t) {
  const int nt = t % p.tn, mt = t / p.tn;
  const int xt = mt % p.tx, yt = (mt / p.tx) % p.ty, bt = mt / (p.tx * p.ty);
  return TileCoord{xt * p.bw, yt * p.bh, bt * p.bb, nt * CT_BN};
}

// rows r, r + 8 of one 64-row accumulator fragment (column pair cq of every 8-column block) -> out, in the fp32 kernel's order:
// (acc + bias) + residual
__device__ __forceinline__ void store_rows(const ConvTcArgs& p, const TileCoord& tc_, int r, int cq, int box_px, const float (&acc)[64]) {
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

__device__ __forceinline__ uint32_t f16x2_rn(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// The A fragments of one k-block for F16Ops, rounded to fp16 from the staged fp32 tile (SWIZZLE_128B, one pixel per 128-byte row):
// af[8 h + 4 k + i] is register i of the m64k16 fragment of pixels 64 h .. 64 h + 63 and channels 16 k .. 16 k + 15, i.e. rows r0 + 8 (i & 1)
// and channel pair 2 t4 + 8 (i >> 1).  A warp's float2 reads of one register cover 8 rows x 2 chunks, 32 distinct banks per 128 bytes.
__device__ __forceinline__ void load_a_f16(const uint8_t* a, int r0, int t4, uint32_t (&af)[16]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = 64 * h + r0 + 8 * (i & 1);
        const float2 v = *reinterpret_cast<const float2*>(a + tc::sw128_offset(row, 4 * k + 2 * (i >> 1) + (t4 >> 1)) + 8 * (t4 & 1));
        af[8 * h + 4 * k + i] = f16x2_rn(v.x, v.y);
      }
}

__device__ __forceinline__ void wgmma_kblock_f16(float (&acc0)[64], float (&acc1)[64], const uint32_t (&af)[16], uint64_t bd) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const uint32_t a0[4] = {af[4 * k], af[4 * k + 1], af[4 * k + 2], af[4 * k + 3]};
    const uint32_t a1[4] = {af[8 + 4 * k], af[9 + 4 * k], af[10 + 4 * k], af[11 + 4 * k]};
    tc::wgmma_128_rs_f16(acc0, a0, bd + 2ull * k, 1u);
    tc::wgmma_128_rs_f16(acc1, a1, bd + 2ull * k, 1u);
  }
}

// The tile loop of gemm_wg_kernel (tc_kernels.cu): warp 8 streams the k-blocks of the CTA's tiles through one ring, the two MMA
// warpgroups take alternate tiles and hand the MMA issue to each other with BAR_TURN.  The epilogue adds bias and residual to the
// accumulator fragments and stores the pixels inside the image straight to global memory (a quad of threads writes 8 consecutive
// channels of a pixel).
template <int KS, class Op>
__global__ void __launch_bounds__(CT_THREADS, 1) unet_conv_tc_kernel(const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm2,
                                                                     const __grid_constant__ CUtensorMap tmw, const ConvTcArgs p) {
  constexpr bool F16 = Op::B_ELEM == 2;
  constexpr int S = Op::STAGES, STAGE_BYTES = ConvTc<Op>::STAGE_BYTES;
  KDB_PDL_TRIGGER();
  uint8_t* base = tc::smem_1k();
  auto* ring = reinterpret_cast<tc::TmaRing<S>*>(base + S * STAGE_BYTES);
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
              const auto ps = PipeState<S>::at(it);
              uint64_t* bar = ring->acquire(ps, STAGE_BYTES);
              uint8_t* a = base + (size_t)ps.slot * STAGE_BYTES;
              if constexpr (F16) {
                const int sh = s ? p.shift2 : 0;
                tc::tma_load_4d(a, s ? &tm2 : &tm1, bar, cb * CT_BK - sh, tc_.x0 + dx, tc_.y0 + dy, tc_.b0);
                tc::tma_load_3d(a + CT_A_BYTES, &tmw, bar, (s ? p.c1 - sh : 0) + cb * CT_BK, tap, tc_.n0);
              } else {
                tc::tma_load_4d(a, s ? &tm2 : &tm1, bar, cb * CT_BK, tc_.x0 + dx, tc_.y0 + dy, tc_.b0);
                tc::tma_load_3d(a + CT_A_BYTES, &tmw, bar, (s ? p.c1 : 0) + cb * CT_BK, tap, tc_.n0);
              }
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
    // one k-block: wait for its stage, issue its MMAs (F16Ops: with A converted into af), and once k-block kb - 1 has completed, release
    // that stage
    auto kblock = [&](int kb, uint32_t(&af)[16]) {
      const auto ps = PipeState<S>::at(it0 + kb);
      ring->wait(ps);
      const uint32_t a_addr = tc::smem_u32(base + (size_t)ps.slot * STAGE_BYTES);
      if constexpr (F16) {
        const uint64_t bd = tc::smem_desc_k_sw64(a_addr + CT_A_BYTES);
        load_a_f16(base + (size_t)ps.slot * STAGE_BYTES, r0, lane & 3, af);
        tc::wg_fence_acc(acc0);
        tc::wg_fence_acc(acc1);
        tc::wg_fence_acc(af);
        tc::wg_fence();
        wgmma_kblock_f16(acc0, acc1, af, bd);
      } else {
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
      }
      tc::wg_commit();
      tc::wg_wait<1>();                  // k-block kb - 1 has completed: its stage (and its A fragments) may be refilled
      tc::wg_fence_acc(acc0);
      tc::wg_fence_acc(acc1);
      if constexpr (F16) tc::wg_fence_acc(af);
      if (kb > 0 && lane == 0) ring->release(PipeState<S>::at(it0 + kb - 1));
    };
    // F16Ops: the A fragments of consecutive k-blocks alternate between afe and afo.  While the wgmmas of one k-block read one set, the
    // next k-block is converted into the other, which the k-block before has finished with.
    uint32_t afe[16], afo[16];
    if constexpr (F16) {
      int kb = 0;
      for (; kb + 1 < nkb; kb += 2) {
        kblock(kb, afe);
        kblock(kb + 1, afo);
      }
      if (kb < nkb) kblock(kb, afe);
    } else {
      for (int kb = 0; kb < nkb; ++kb) kblock(kb, afe);
    }
    if (i + 1 < n_local) tc::named_barrier_arrive(tc::BAR_TURN + (wg ^ 1), 256);
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    if constexpr (F16) {
      tc::wg_fence_acc(afe);
      tc::wg_fence_acc(afo);
    }
    if (lane == 0) ring->release(PipeState<S>::at(it0 + nkb - 1));

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

__global__ void __launch_bounds__(256) round_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, int64_t rows, int C, int ld) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows * ld; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld;
    const int c = (int)(i - r * ld);
    dst[i] = c < C ? __float2half_rn(src[r * C + c]) : __float2half_rn(0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// global self-attention (SelfAttention2d, layers.py:181-200), d_head 64, on mma.sync: m16n8k8 tf32 (Tf32Ops) or m16n8k16 fp16 (F16Ops)
// ------------------------------------------------------------------------------------------------
// A CTA of 4 warps takes 64 queries of one (image, head); each warp owns 16 of them.  The CTA walks the keys in blocks of 64: K and V
// of the block are staged in shared memory (stage_kv), S = Q K^T is a register fragment, the softmax keeps a running maximum per row (q
// and k are not normalised: no logit bound) and rescales O and l when it grows (RunningSoftmax), and O += P V takes P straight from the
// S fragment.
//
// Tf32Ops: K and V rows of 68 floats (the fragment reads of both hit 32 distinct banks).  No transpose of V is needed: the B operand of
// mma.sync is loaded per thread from registers, and the k index of the P V product is relabelled inside each 8-key group (A column t
// <-> key 2t, column t + 4 <-> key 2t + 1), so the accumulator pair a thread holds of S is exactly its A fragment of P, and V is read at
// the matching keys.  q, k, v and P are truncated to tf32 (low 13 bits cleared) like the convolution's activations.
//
// F16Ops: K and V rows of 72 fp16, rounded to nearest even as they are staged (144-byte rows: the K fragment reads and the ldmatrix
// rows hit 32 distinct banks).  The two S accumulators of 8-key groups 2jj and 2jj + 1 are, packed to fp16 pairs, the thread's A
// fragment of P for keys 16jj .. 16jj + 15 in the natural order; V's B fragment along keys comes from ldmatrix.trans of the staged
// [key][d] rows.  q, k, v and P are rounded to fp16.
//
// Both: l sums the rounded P.
constexpr int AT_D = 64, AT_Q = 64, AT_KB = 64, AT_THREADS = 128;
template <class Op>
struct AttnTc;
template <>
struct AttnTc<Tf32Ops> {
  using Elem = float;
  static constexpr int LD = 68;
};
template <>
struct AttnTc<F16Ops> {
  using Elem = __half;
  static constexpr int LD = 72;
};
template <class Op>
constexpr size_t at_smem() {
  return (size_t)2 * AT_KB * AttnTc<Op>::LD * sizeof(typename AttnTc<Op>::Elem);
}

__device__ __forceinline__ uint32_t tf32_bits(float v) { return __float_as_uint(v) & 0xffffe000u; }

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void store4(float* dst, float4 v) { *reinterpret_cast<float4*>(dst) = v; }
__device__ __forceinline__ void store4(__half* dst, float4 v) { *reinterpret_cast<uint2*>(dst) = make_uint2(f16x2_rn(v.x, v.y), f16x2_rn(v.z, v.w)); }

// K and V rows of the key block at k0 -> Ks, Vs ([AT_KB][LD] elements), zeros past the T keys
template <int LD, class E>
__device__ __forceinline__ void stage_kv(const float* base, int C, int head, int k0, int T, E* Ks, E* Vs) {
  for (int i = threadIdx.x; i < AT_KB * AT_D / 4; i += AT_THREADS) {
    const int r = i / (AT_D / 4), c4 = (i % (AT_D / 4)) * 4;
    float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
    if (k0 + r < T) {
      const float* row = base + (int64_t)(k0 + r) * 3 * C + head * AT_D + c4;
      kv = *reinterpret_cast<const float4*>(row + C);
      vv = *reinterpret_cast<const float4*>(row + 2 * C);
    }
    store4(Ks + r * LD + c4, kv);
    store4(Vs + r * LD + c4, vv);
  }
}

constexpr float LOG2E = 1.4426950408889634f;

// Running-maximum softmax of the rows g (entries 0, 1 of each S fragment) and g + 8 (entries 2, 3) of a thread's quad
struct RunningSoftmax {
  float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // masks the keys past T of the 64-key block at k0, raises the maxima and rescales O and l; -> mb0, mb1: the maxima times log2(e)
  __device__ __forceinline__ void update(float (&sf)[8][4], int k0, int t4, int T, float (&o)[8][4], float& mb0, float& mb1) {
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
    mb0 = n0 * LOG2E;
    mb1 = n1 * LOG2E;
  }

  // the unnormalised probability of score s in a row whose maximum times log2(e) is mb
  static __device__ __forceinline__ float p(float s, float mb) { return exp2f(fmaf(s, LOG2E, -mb)); }

  // O / l of the rows q0 + g, q0 + 8 + g that exist -> out (row stride C)
  __device__ __forceinline__ void store(float* out, int T, int q0, int g, int t4, int C, const float (&o)[8][4]) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + g + 8 * h;
      if (q >= T) continue;
      float* orow = out + (int64_t)q * C;
#pragma unroll
      for (int n = 0; n < 8; ++n)
        *reinterpret_cast<float2*>(orow + 8 * n + 2 * t4) = make_float2(o[n][2 * h] * (h ? inv1 : inv0), o[n][2 * h + 1] * (h ? inv1 : inv0));
    }
  }
};

template <class Op>
__global__ void __launch_bounds__(AT_THREADS) unet_attn_tc_kernel(const float* __restrict__ qkv, float* __restrict__ out, int T, int nh) {
  constexpr bool F16 = std::is_same<Op, F16Ops>::value;
  using E = typename AttnTc<Op>::Elem;
  constexpr int LD = AttnTc<Op>::LD;
  extern __shared__ __align__(16) uint8_t at_sm[];
  E* Ks = reinterpret_cast<E*>(at_sm);     // [AT_KB][LD]
  E* Vs = Ks + AT_KB * LD;
  const int head = blockIdx.y, b = blockIdx.z, C = nh * AT_D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int q0 = blockIdx.x * AT_Q + warp * 16;
  const float* base = qkv + (int64_t)b * T * 3 * C;
  // Q A fragments along d, rows g, g + 8: tf32, 8 k-steps of columns t4, t4 + 4; fp16, 4 k-steps of column pairs 2 t4, 2 t4 + 8
  uint32_t qa[8][4];
#pragma unroll
  for (int kk = 0; kk < (F16 ? 4 : 8); ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = q0 + g + 8 * (i & 1);
      const float* qr = base + (int64_t)q * 3 * C + head * AT_D;
      if constexpr (F16) {
        const int d = 16 * kk + 2 * t4 + 8 * (i >> 1);
        qa[kk][i] = q < T ? f16x2_rn(qr[d], qr[d + 1]) : 0u;
      } else {
        const int d = 8 * kk + t4 + 4 * (i >> 1);
        qa[kk][i] = q < T ? tf32_bits(qr[d]) : 0u;
      }
    }
  float o[8][4];
  RunningSoftmax sm;
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  for (int k0 = 0; k0 < T; k0 += AT_KB) {
    __syncthreads();                       // the previous block's K / V are no longer read
    stage_kv<LD>(base, C, head, k0, T, Ks, Vs);
    __syncthreads();
    // S = Q K^T for 64 keys: 8 fragments of 8 keys
    float sf[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sf[j][0] = sf[j][1] = sf[j][2] = sf[j][3] = 0.f;
      const E* kr = Ks + (8 * j + g) * LD;
      if constexpr (F16) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          mma_f16(sf[j], qa[kk], *reinterpret_cast<const uint32_t*>(kr + 16 * kk + 2 * t4),
                  *reinterpret_cast<const uint32_t*>(kr + 16 * kk + 2 * t4 + 8));
      } else {
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          mma_tf32(sf[j], qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], tf32_bits(kr[8 * kk + t4]), tf32_bits(kr[8 * kk + t4 + 4]));
      }
    }
    float mb0, mb1;
    sm.update(sf, k0, t4, T, o, mb0, mb1);
    if constexpr (F16) {
      // P (rounded to fp16) and O += P V, one 16-key group per k-step
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        uint32_t pa[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // e: rows g (0, 2), g + 8 (1, 3); keys 16 jj + 2 t4 (0, 1), + 8 (2, 3)
          const float* s2 = sf[2 * jj + (e >> 1)] + 2 * (e & 1);
          const float mb = (e & 1) ? mb1 : mb0;
          pa[e] = f16x2_rn(RunningSoftmax::p(s2[0], mb), RunningSoftmax::p(s2[1], mb));
          const float2 pr = __half22float2(*reinterpret_cast<const __half2*>(&pa[e]));
          if (e & 1) sm.l1 += pr.x + pr.y;
          else sm.l0 += pr.x + pr.y;
        }
        // lane l addresses row (l & 7) of matrix l >> 3: keys 16 jj + {0-7, 8-15} x d {0-7, 8-15} of each 16-column pair np
        const uint32_t vrow = tc::smem_u32(Vs + (16 * jj + (lane & 7) + 8 * ((lane >> 3) & 1)) * LD + 8 * (lane >> 4));
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          uint32_t v0, v1, v2, v3;
          asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                       : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3)
                       : "r"(vrow + 32u * np));
          mma_f16(o[2 * np], pa, v0, v1);
          mma_f16(o[2 * np + 1], pa, v2, v3);
        }
      }
    } else {
      // P (truncated to tf32) and O += P V, one 8-key group per k-step
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t p[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          p[e] = tf32_bits(RunningSoftmax::p(sf[j][e], (e >> 1) ? mb1 : mb0));
          if (e >> 1) sm.l1 += __uint_as_float(p[e]);
          else sm.l0 += __uint_as_float(p[e]);
        }
        const float* v0 = Vs + (8 * j + 2 * t4) * LD;   // keys 8j + 2 t4 (A column t4) and + 1 (A column t4 + 4)
#pragma unroll
        for (int n = 0; n < 8; ++n) mma_tf32(o[n], p[0], p[2], p[1], p[3], tf32_bits(v0[8 * n + g]), tf32_bits(v0[LD + 8 * n + g]));
      }
    }
  }
  sm.store(out + (int64_t)b * T * C + head * AT_D, T, q0, g, t4, C, o);
}

int pow2_at_least(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// [B, H, W, C] fp32 tokens as the 4-D map (C, W, H, B) with the tile's pixel box
int tmap_tokens_f32(CUtensorMap* t, const float* base, int C, const ConvArgs& a, const ConvTcArgs& p) {
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.B};
  const uint64_t strides[3] = {(uint64_t)C * 4, (uint64_t)C * 4 * a.W, (uint64_t)C * 4 * a.W * a.H};
  const uint32_t box[4] = {CT_BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bb};
  return make_tmap_f32(t, base, 4, dims, strides, box);
}

template <int KS, class Op>
int launch_conv_tc(const CUtensorMap& t1, const CUtensorMap& t2, const CUtensorMap& tw, const ConvTcArgs& p, int64_t tiles, cudaStream_t st) {
  static bool opened = false;
  int rc;
  if ((rc = set_smem_once(unet_conv_tc_kernel<KS, Op>, opened, (int)ConvTc<Op>::SMEM))) return rc;
  KDB_CUDA(launch_pdl(unet_conv_tc_kernel<KS, Op>, persistent_grid(tiles), dim3(CT_THREADS), ConvTc<Op>::SMEM, st, t1, t2, tw, p));
  return 0;
}

// the convolution at either operand format: w is the tf32-rounded fp32 weight [N, ks*ks, c1 + c2] (Tf32Ops) or the fp16 weight
// [N, ks*ks, f16_weight_ld(c1 + c2)] (F16Ops)
template <class Op>
int launch_conv_tc(const ConvArgs& a, const void* w, int ks, cudaStream_t st, const char* name, int family) {
  KDB_REQUIRE(ks == 1 || ks == 3, KDB_ERR_BAD_ARG, "%s: kernel size %d", name, ks);
  KDB_REQUIRE(a.in1 && w && a.out && a.B > 0 && a.H > 0 && a.W > 0 && a.N > 0 && a.c1 > 0, KDB_ERR_BAD_ARG, "%s: bad arguments", name);
  KDB_REQUIRE(a.c2 == 0 || a.in2, KDB_ERR_BAD_ARG, "%s: %d channels of a second source without its pointer", name, a.c2);
  KDB_REQUIRE(a.c1 % 4 == 0 && a.c2 % 4 == 0 && a.rc1 % 4 == 0, KDB_ERR_BAD_SHAPE, "%s: channel counts %d + %d must be multiples of 4", name,
              a.c1, a.c2);
  KDB_REQUIRE(!a.r1 || a.rc1 == a.N || (a.r2 && a.rc1 < a.N), KDB_ERR_BAD_ARG, "%s: bad residual split", name);
  ConvTcArgs p{};
  p.bias = a.bias, p.r1 = a.r1, p.r2 = a.r2, p.out = a.out;
  p.rc1 = a.rc1, p.N = a.N, p.B = a.B, p.H = a.H, p.W = a.W, p.c1 = a.c1;
  p.shift2 = std::is_same<Op, F16Ops>::value && a.c2 ? a.c1 % 8 : 0;
  p.kb1 = (int)ceil_div(a.c1, CT_BK), p.kb2 = (int)ceil_div(a.c2 + p.shift2, CT_BK);
  p.bw = std::min(pow2_at_least(a.W), CT_BM);
  p.bh = std::min(pow2_at_least(a.H), CT_BM / p.bw);
  p.bb = CT_BM / (p.bw * p.bh);
  p.tx = (int)ceil_div(a.W, p.bw), p.ty = (int)ceil_div(a.H, p.bh), p.tn = (int)ceil_div(a.N, CT_BN);
  const int64_t tiles = (int64_t)p.tx * p.ty * ceil_div(a.B, p.bb) * p.tn;
  KDB_REQUIRE(tiles <= (1ll << 30), KDB_ERR_BAD_SHAPE, "%s: %lld tiles", name, (long long)tiles);
  CUtensorMap t1, t2, tw;
  int rc;
  if ((rc = tmap_tokens_f32(&t1, a.in1, a.c1, a, p))) return rc;
  if ((rc = tmap_tokens_f32(&t2, a.c2 ? a.in2 : a.in1, a.c2 ? a.c2 : a.c1, a, p))) return rc;
  const int Ct = a.c1 + a.c2;
  const uint64_t ld = std::is_same<Op, F16Ops>::value ? (uint64_t)f16_weight_ld(Ct) * 2 : (uint64_t)Ct * 4;   // bytes per weight row
  const uint64_t wdims[3] = {(uint64_t)Ct, (uint64_t)(ks * ks), (uint64_t)a.N};
  const uint64_t wstrides[2] = {ld, ld * ks * ks};
  const uint32_t wbox[3] = {CT_BK, 1, CT_BN};
  if ((rc = std::is_same<Op, F16Ops>::value ? make_tmap_f16_sw64(&tw, w, 3, wdims, wstrides, wbox)
                                            : make_tmap_f32(&tw, w, 3, wdims, wstrides, wbox)))
    return rc;
  if ((rc = ks == 3 ? launch_conv_tc<3, Op>(t1, t2, tw, p, tiles, st) : launch_conv_tc<1, Op>(t1, t2, tw, p, tiles, st))) return rc;
  KDB_LAUNCH_CHECK(family, st);
  return 0;
}

template <class Op>
int launch_attn_tc(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st, const char* name, int family) {
  KDB_REQUIRE(qkv && out && B > 0 && T > 0 && nh > 0, KDB_ERR_BAD_ARG, "%s: bad arguments", name);
  KDB_REQUIRE(unet_attn_tc_supported(d_head), KDB_ERR_UNSUPPORTED, "%s: d_head %d (the kernel is built for 64)", name, d_head);
  KDB_REQUIRE(B <= 65535 && nh <= 65535, KDB_ERR_BAD_SHAPE, "%s: %d images x %d heads exceed the grid", name, B, nh);
  unet_attn_tc_kernel<Op><<<dim3((unsigned)ceil_div(T, AT_Q), (unsigned)nh, (unsigned)B), AT_THREADS, at_smem<Op>(), st>>>(qkv, out, T, nh);
  KDB_LAUNCH_CHECK(family, st);
  return 0;
}

}  // namespace

int f16_weight_ld(int channels) { return (channels + 7) / 8 * 8; }

int launch_unet_conv_tf32(const ConvArgs& a, int ks, cudaStream_t st, int family) {
  return launch_conv_tc<Tf32Ops>(a, a.w, ks, st, "unet_conv_tf32", family);
}

int launch_unet_conv_fp16(const ConvArgs& a, const __half* w, int ks, cudaStream_t st) {
  return launch_conv_tc<F16Ops>(a, w, ks, st, "unet_conv_fp16", F_UNET_CONV_FP16);
}

bool unet_attn_tc_supported(int d_head) { return d_head == AT_D; }

int launch_unet_attn_tf32(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st) {
  return launch_attn_tc<Tf32Ops>(qkv, out, B, T, nh, d_head, st, "unet_attn_tf32", F_UNET_ATTN_TF32);
}

int launch_unet_attn_fp16(const float* qkv, float* out, int B, int T, int nh, int d_head, cudaStream_t st) {
  return launch_attn_tc<F16Ops>(qkv, out, B, T, nh, d_head, st, "unet_attn_fp16", F_UNET_ATTN_FP16);
}

int launch_unet_round_tf32(const float* src, float* dst, int64_t n, cudaStream_t st) {
  round_tf32_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), (int64_t)kNumSMs * 32), 256, 0, st>>>(src, dst, n);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

int launch_unet_round_f16(const float* src, __half* dst, int64_t rows, int C, cudaStream_t st) {
  const int ld = f16_weight_ld(C);
  round_f16_kernel<<<(unsigned)std::min<int64_t>(ceil_div(rows * ld, 256), (int64_t)kNumSMs * 32), 256, 0, st>>>(src, dst, rows, C, ld);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

}  // namespace kdb
