// tc_kernels.cu -- bf16 tensor-core GEMM for sm_90a: TMA (SWIZZLE_128B tiles) -> shared memory -> wgmma (fp32 accumulators in
// registers) -> fp32 shared-memory tile -> fused epilogue (thread = output row) -> swizzled shared tile -> TMA store.
//
// C[M,N] = A[M,K] W[N,K]^T for every nn.Linear on the token stream (reference image_transformer_v2.py:126-139).
// Epilogues: plain store; +residual (out_proj / down_proj, :396,:493; residual tile prefetched by TMA while the main loop
// runs); GEGLU (:89-95; rows of W interleaved 8 value / 8 gate); cosine-sim scaling + axial RoPE of q and k fused into the
// qkv projection (:106-114,187-199,245-248; cos/sin from a per-layer table); TokenSplit scatter + lerp (:618-621).
//
// Warp roles in a 160-thread CTA: warps 0-3 = the warpgroup that issues wgmma and then runs the epilogue (one accumulator row
// per thread), warp 4 = TMA producer (one elected lane).  One 128 x BN output tile per CTA; two CTAs are co-resident per SM so
// one tile's epilogue overlaps the other's main loop.  Output rows are written to a SWIZZLE_128B staging tile and leave through
// one TMA store per 64 columns: fully coalesced, clipped at the M edge by the tensor map.
#include "tc_common.cuh"
#include "tc_kernels.cuh"

namespace kdb {

// ------------------------------------------------------------------------------------------------
// tensor maps (driver entry point fetched through the runtime: no link-time libcuda dependency)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = encode_fn();
  KDB_REQUIRE(fn != nullptr, KDB_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled not available from this driver");
  cuuint64_t gd[5];
  cuuint64_t gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gs[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  KDB_REQUIRE(r == CUDA_SUCCESS, KDB_ERR_BAD_ARG, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dim0 %llu, box0 %u)", (int)r,
              rank, (unsigned long long)dims[0], box[0]);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int BM = 128, BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KiB
constexpr int SUB_TILE_BYTES = BM * 128;     // one [128 x 64] bf16 output sub-tile
constexpr int MAX_STAGES = 4;
constexpr int GEMM_THREADS = 160;            // warps 0-3: MMA + epilogue warpgroup, warp 4: TMA producer

enum TcEpi { TCE_STORE = 0, TCE_RESID = 1, TCE_GEGLU = 2, TCE_SPLIT = 3, TCE_QKV = 4, TCE_PATCHOUT = 5 };

struct TcParams {
  bf16* out;
  const bf16* resid;     // SPLIT: skip [B, 2hc, 2wc, Cf]
  const float* fac;
  int64_t M;
  int N, K, stages;
  int hc, wc, Cf;
  // QKV
  const float2* rope;    // float4 [nh][8][T] (cos, cos, sin, sin) of angle pairs, see rope_table_kernel
  const float* qk_scale; // [nh]
  int C, nh, T;
  // PATCHOUT (4x4 patches, 3 output channels): un-patch to NCHW fp32 + Karras combine with the input latent
  float* fout;
  const float* x_in;
  const float* sigma;
  float sd;
  int H, Wimg, th, tw;
  const float* ss_in;    // fused RMSNorm (consumer): A = raw x, W carries the channel scale; [M, SS_PARTS] sums of squares of x
  float* ss_out;         // RESID / SPLIT / STORE (producer): sums of squares of the rows written, for the next fused RMSNorm
  int a_merge, mwc, mC;  // A operand gathered from fine tokens (TokenMerge): coarse grid width, fine channels
  int box_w, box_h;      // 5-D TMA box of the merge gather: 128 rows = box_h x box_w coarse tokens
};

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

int tmap_2d(CUtensorMap* t, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer) {
  const uint64_t dims[2] = {inner, outer};
  const uint64_t strides[1] = {inner * 2};
  const uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_bf16(t, base, 2, dims, strides, box);
}

// 5-D view of a fine token tensor X[B, 2*hc, 2*wc, C] as (e, nw, wx, nh, b*hc+hy): one (nh, nw) quadrant of `box_h x box_w`
// coarse tokens x 64 channels is a [128 x 64] SWIZZLE_128B tile in coarse-token order -- TokenMerge's gather becomes TMA
// coordinates (reference image_transformer_v2.py:594,607).
int tmap_quad(CUtensorMap* t, const void* base, int C, int wc, uint64_t bhc, int box_w, int box_h) {
  const uint64_t dims[5] = {(uint64_t)C, 2, (uint64_t)wc, 2, bhc};
  const uint64_t strides[4] = {(uint64_t)C * 2, (uint64_t)C * 4, (uint64_t)wc * C * 4, (uint64_t)wc * C * 8};
  const uint32_t box[5] = {64, 1, (uint32_t)box_w, 1, (uint32_t)box_h};
  return make_tmap_bf16(t, base, 5, dims, strides, box);
}

// 128 consecutive coarse tokens as a box_h x box_w rectangle of the coarse grid (rows of width wc)
bool quad_box(int wc, int* box_w, int* box_h) {
  if (wc >= BM) {
    if (wc % BM != 0) return false;
    *box_w = BM;
    *box_h = 1;
    return true;
  }
  if (BM % wc != 0) return false;
  *box_w = wc;
  *box_h = BM / wc;
  return true;
}

// Shared memory of one GEMM CTA: the TMA ring, which the fp32 accumulator tile re-uses once the main loop is done, then the bf16
// output staging tile (RESID: the residual tile is loaded into it and the epilogue adds in place), then the barriers.
template <int BN> constexpr int acc_ld() { return BN + 4; }   // fp32 accumulator row pitch (+4: rows start on different banks)
template <int BN, int EPI> constexpr int out_bytes() {
  return EPI == TCE_GEGLU ? SUB_TILE_BYTES : (EPI == TCE_SPLIT || EPI == TCE_PATCHOUT) ? 0 : (BN / 64) * SUB_TILE_BYTES;
}
template <int BN>
__host__ __device__ inline size_t gemm_region0(int stages) {
  const size_t ring = (size_t)stages * (A_STAGE_BYTES + BN * BK * 2), acc = (size_t)BM * acc_ld<BN>() * 4;
  return ((ring > acc ? ring : acc) + 1023) & ~(size_t)1023;
}
template <int BN, int EPI> inline size_t gemm_smem(int stages) { return 1024 + gemm_region0<BN>(stages) + out_bytes<BN, EPI>() + 128; }

// C[M,N] tile of 128 x BN per CTA.  Warp 4 (one elected lane) streams A / W k-blocks through a ring of SWIZZLE_128B stages; the
// warpgroup of warps 0-3 issues wgmma (two M = 64 halves per k-step) with the accumulators in registers, keeps one k-block in
// flight while it releases the previous stage, then writes the accumulators to an fp32 tile in shared memory so that each thread
// owns one output row for the fused epilogue (fp32 arithmetic, one rounding to bf16 at the pack, one TMA store per 64 columns).
template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS) gemm_wg_kernel(const __grid_constant__ CUtensorMap tma, const __grid_constant__ CUtensorMap tmb,
                                                               const __grid_constant__ CUtensorMap tmc, const __grid_constant__ CUtensorMap tmr,
                                                               const TcParams p) {
  KDB_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  constexpr int NSUB = BN / 64;
  constexpr int LD = acc_ld<BN>();
  constexpr bool RES = EPI == TCE_RESID;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* sAcc = reinterpret_cast<float*>(base);
  uint8_t* sC = base + gemm_region0<BN>(p.stages);
  uint64_t* full = reinterpret_cast<uint64_t*>(sC + out_bytes<BN, EPI>());
  uint64_t* empty = full + MAX_STAGES;
  uint64_t* resid_full = empty + MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int nkb = p.K / BK;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tma);
    tc::tma_prefetch_desc(&tmb);
    for (int s = 0; s < p.stages; ++s) {
      tc::mbar_init(&full[s], 1);
      tc::mbar_init(&empty[s], 4);       // lane 0 of each MMA warp
    }
    tc::mbar_init(resid_full, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      if constexpr (RES) {
        tc::mbar_arrive_expect_tx(resid_full, NSUB * SUB_TILE_BYTES);
#pragma unroll
        for (int g = 0; g < NSUB; ++g) tc::tma_load_2d(sC + g * SUB_TILE_BYTES, &tmr, resid_full, n0 + g * 64, (int)m0);
      }
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % p.stages;
        const uint32_t ph = (uint32_t)(kb / p.stages) & 1u;
        tc::mbar_wait(&empty[s], ph ^ 1u);
        tc::mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
        uint8_t* a = base + (size_t)s * STAGE_BYTES;
        if (p.a_merge) {   // TokenMerge: k-block kb lives in quadrant (nh, nw) of the fine grid, channels e0..e0+63
          const int qd = (kb * BK) / p.mC, e0 = kb * BK - qd * p.mC;
          tc::tma_load_5d(a, &tma, &full[s], e0, qd & 1, p.box_h == 1 ? (int)(m0 % p.mwc) : 0, qd >> 1, (int)(m0 / p.mwc));
        } else {
          tc::tma_load_2d(a, &tma, &full[s], kb * BK, (int)m0);
        }
        tc::tma_load_2d(a + A_STAGE_BYTES, &tmb, &full[s], kb * BK, n0);
      }
    }
    return;
  }

  // ---------------- main loop: warpgroup MMA, accumulators in registers
  {
    float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % p.stages;
      tc::mbar_wait(&full[s], (uint32_t)(kb / p.stages) & 1u);
      const uint32_t a_addr = tc::smem_u32(base + (size_t)s * STAGE_BYTES);
      const uint64_t ad0 = tc::smem_desc_k_sw128(a_addr), ad1 = tc::smem_desc_k_sw128(a_addr + 8 * 1024);   // rows 0-63 / 64-127
      const uint64_t bd = tc::smem_desc_k_sw128(a_addr + A_STAGE_BYTES);
      tc::wg_fence_acc(acc0);
      tc::wg_fence_acc(acc1);
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {   // advance 16 bf16 = 32 B along K inside the swizzle atom: +2 in the (addr >> 4) field
        if constexpr (BN == 128) {
          tc::wgmma_128(acc0, ad0 + 2ull * k, bd + 2ull * k, 1u);
          tc::wgmma_128(acc1, ad1 + 2ull * k, bd + 2ull * k, 1u);
        } else {
          tc::wgmma_64<0>(acc0, ad0 + 2ull * k, bd + 2ull * k, 1u);
          tc::wgmma_64<0>(acc1, ad1 + 2ull * k, bd + 2ull * k, 1u);
        }
      }
      tc::wg_commit();
      tc::wg_wait<1>();                  // k-block kb - 1 has completed: its stage may be refilled
      tc::wg_fence_acc(acc0);
      tc::wg_fence_acc(acc1);
      if (kb > 0 && lane == 0) tc::mbar_arrive(&empty[(kb - 1) % p.stages]);
    }
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    tc::named_barrier_sync(1, 128);      // every read of the ring is done: the accumulator tile may overwrite it
    tc::acc_store(sAcc, LD, 0, acc0);
    tc::acc_store(sAcc, LD, 64, acc1);
  }
  tc::named_barrier_sync(1, 128);

  // ---------------- epilogue: thread = output row
  const int row = threadIdx.x;
  const int64_t m = m0 + row;
  float rstd = 1.f;
  if (p.ss_in != nullptr) {   // fused RMSNorm (consumer side): the producer of x left sum(x^2) of every token, one slot per 128 channels
    const float4* sp = reinterpret_cast<const float4*>(p.ss_in + (m < p.M ? m : 0) * SS_PARTS);
    rstd = rsqrtf(tc::rowss_sum(__ldg(sp), __ldg(sp + 1), p.K >> 7) / (float)p.K + 1e-6f);
  }
  if constexpr (EPI == TCE_PATCHOUT) {
    // TokenSplitWithoutSkip 4x4 + NCHW + Denoiser combine (reference :598-607,:758-760, layers.py:88-90).  Row m = token
    // (b, ty, tx); column n = (nh*4 + nw)*3 + c.  For fixed (c, nh) the 4 nw pixels are one float4.
    float v[64];
    {
      float t0[32], t1[32];
      tc::acc_ld32(sAcc, LD, row, 0, t0);
      tc::acc_ld32(sAcc, LD, row, 32, t1);
#pragma unroll
      for (int i = 0; i < 32; ++i) { v[i] = t0[i]; v[32 + i] = t1[i]; }
    }
    if (m < p.M) {
      if (p.ss_in != nullptr) {   // fused out_norm: A is the raw residual stream, W carries the channel scale
#pragma unroll
        for (int i = 0; i < 48; ++i) v[i] *= rstd;
      }
      const int per = p.th * p.tw;
      const int b = (int)(m / per);
      const int r = (int)(m - (int64_t)b * per);
      const int ty = r / p.tw, tx = r - ty * p.tw;
      float c_skip = 0.f, c_out = 1.f, c_in;
      if (p.sd > 0.f) karras_scalings(__ldg(p.sigma + b), p.sd, c_skip, c_out, c_in);
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int nh = 0; nh < 4; ++nh) {
          const int64_t o = (((int64_t)b * 3 + c) * p.H + (ty * 4 + nh)) * p.Wimg + tx * 4;
          float4 y = make_float4(bf16_round(v[(nh * 4 + 0) * 3 + c]), bf16_round(v[(nh * 4 + 1) * 3 + c]), bf16_round(v[(nh * 4 + 2) * 3 + c]),
                                 bf16_round(v[(nh * 4 + 3) * 3 + c]));
          if (p.sd > 0.f) {
            const float4 xi = __ldg(reinterpret_cast<const float4*>(p.x_in + o));
            y = make_float4(y.x * c_out + xi.x * c_skip, y.y * c_out + xi.y * c_skip, y.z * c_out + xi.z * c_skip, y.w * c_out + xi.w * c_skip);
          }
          *reinterpret_cast<float4*>(p.fout + o) = y;
        }
    }
  } else if constexpr (EPI == TCE_SPLIT) {
    // TokenSplit + torch.lerp(skip, x, fac) (reference :618-621): row m = (b, hy, wx) on the coarse grid; 32 columns inside one
    // (nh, nw) quadrant (Cf % 32 == 0), scattered to the fine token
    const bool live = m < p.M;
    const float facv = __ldg(p.fac);
    float ss = 0.f;
    int64_t fine = 0;
#pragma unroll 1
    for (int c = 0; c < BN / 32; ++c) {
      float v[32];
      tc::acc_ld32(sAcc, LD, row, c * 32, v);
      if (!live) continue;
      const int n = n0 + c * 32;
      const int64_t b = m / ((int64_t)p.hc * p.wc);
      const int r = (int)(m - b * p.hc * p.wc);
      const int hy = r / p.wc, wx = r - hy * p.wc;
      const int qd = n / p.Cf, e = n - qd * p.Cf;
      fine = (b * (2 * p.hc) + (2 * hy + (qd >> 1))) * (2 * p.wc) + (2 * wx + (qd & 1));
      const int64_t off = fine * p.Cf + e;
      const uint4* sk = reinterpret_cast<const uint4*>(p.resid + off);
      uint4* dst = reinterpret_cast<uint4*>(p.out + off);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 r4 = sk[j];
        const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
        uint32_t ow[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float lo = __uint_as_float(rw[t] << 16), hi = __uint_as_float(rw[t] & 0xffff0000u);   // bf16 -> fp32 is a shift / mask
          const float e0 = v[j * 8 + t * 2], e1 = v[j * 8 + t * 2 + 1];
          const float d0 = e0 - lo, d1 = e1 - hi;
          const float o0 = (facv < 0.5f) ? fmaf(facv, d0, lo) : e0 - d0 * (1.f - facv);
          const float o1 = (facv < 0.5f) ? fmaf(facv, d1, hi) : e1 - d1 * (1.f - facv);
          ss = fmaf(o0, o0, fmaf(o1, o1, ss));
          ow[t] = tc::pack_bf16x2(o0, o1);
        }
        dst[j] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
    }
    // statistics of the new residual stream for the next fused RMSNorm (BN = 128 inside one quadrant: Cf % 128 == 0)
    if (p.ss_out != nullptr && live) p.ss_out[fine * SS_PARTS + ((n0 % p.Cf) >> 7)] = ss;
  } else {
    if constexpr (RES) tc::mbar_wait(resid_full, 0);
    float ss_acc[4] = {0.f, 0.f, 0.f, 0.f};   // producer side: sum of squares of the row this thread writes
#pragma unroll 1
    for (int g = 0; g < NSUB; ++g) {
      float v[64];
      {
        float t0[32], t1[32];
        tc::acc_ld32(sAcc, LD, row, g * 64, t0);
        tc::acc_ld32(sAcc, LD, row, g * 64 + 32, t1);
#pragma unroll
        for (int i = 0; i < 32; ++i) { v[i] = t0[i]; v[32 + i] = t1[i]; }
      }
      if (EPI != TCE_GEGLU && p.ss_in != nullptr) {
        // fused RMSNorm row scale.  q and k are cosine-normalised afterwards (scale invariant): only v needs it.
        bool apply = true;
        if constexpr (EPI == TCE_QKV) apply = (n0 + g * 64) >= 2 * p.C;
        if (apply) {
#pragma unroll
          for (int i = 0; i < 64; ++i) v[i] *= rstd;
        }
      }
      if constexpr (EPI == TCE_GEGLU) {
        // columns come as [8 value | 8 gate] groups (interleaved up_proj rows) -> 32 outputs = chunks 4g..4g+3 of the output sub-tile
        const tc::f32x2 r2 = tc::pk2(rstd, rstd), rh = tc::pk2(0.5f * rstd, 0.5f * rstd);     // the GELU's 0.5 rides on the value's row scale
#pragma unroll
        for (int gg = 0; gg < 4; ++gg) {
          uint32_t o[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            tc::f32x2 val = tc::pk2(v[gg * 16 + 2 * j], v[gg * 16 + 2 * j + 1]);
            tc::f32x2 gate = tc::pk2(v[gg * 16 + 8 + 2 * j], v[gg * 16 + 8 + 2 * j + 1]);
            val = tc::mul2(val, rh);
            if (p.ss_in != nullptr) gate = tc::mul2(gate, r2);
            float o0, o1;
            tc::upk2(tc::geglu2(val, gate), o0, o1);
            o[j] = tc::pack_bf16x2(o0, o1);
          }
          *reinterpret_cast<uint4*>(sC + tc::sw128_offset(row, g * 4 + gg)) = make_uint4(o[0], o[1], o[2], o[3]);
        }
      } else {
        uint8_t* cg = sC + g * SUB_TILE_BYTES;
        if constexpr (RES) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {      // this thread reads and then overwrites only its own row
            const uint4 r4 = *reinterpret_cast<const uint4*>(cg + tc::sw128_offset(row, j));
            const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              v[j * 8 + t * 2] += __uint_as_float(rw[t] << 16);
              v[j * 8 + t * 2 + 1] += __uint_as_float(rw[t] & 0xffff0000u);
            }
          }
        }
        if constexpr (RES || EPI == TCE_STORE) {
          if (p.ss_out != nullptr) {
#pragma unroll
            for (int i = 0; i < 64; i += 4) {
              ss_acc[0] = fmaf(v[i], v[i], ss_acc[0]);
              ss_acc[1] = fmaf(v[i + 1], v[i + 1], ss_acc[1]);
              ss_acc[2] = fmaf(v[i + 2], v[i + 2], ss_acc[2]);
              ss_acc[3] = fmaf(v[i + 3], v[i + 3], ss_acc[3]);
            }
          }
        }
        if constexpr (EPI == TCE_QKV) {
          const int n = n0 + g * 64;               // one head of q, k or v (feature order (t nh e), d_head 64)
          const int t3 = n / p.C, head = (n - t3 * p.C) >> 6;
          if (t3 < 2) {
            // cosine-sim scale + axial RoPE (reference :106-114,187-199,245-248).  Columns (2i, 2i+1) pair with (16+2i, 17+2i); the
            // table holds (cos_2i, cos_2i+1, sin_2i, sin_2i+1) per float4.
            const int64_t tok = (m < p.M ? m : 0) % p.T;
            const float4* tb = reinterpret_cast<const float4*>(p.rope) + (int64_t)head * 8 * p.T + tok;   // [head][i][token]
            tc::f32x2 P[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) P[i] = tc::pk2(v[2 * i], v[2 * i + 1]);
            tc::f32x2 q0 = tc::mul2(P[0], P[0]), q1 = tc::mul2(P[1], P[1]), q2 = tc::mul2(P[2], P[2]), q3 = tc::mul2(P[3], P[3]);
#pragma unroll
            for (int i = 4; i < 32; i += 4) {
              q0 = tc::fma2(P[i], P[i], q0);
              q1 = tc::fma2(P[i + 1], P[i + 1], q1);
              q2 = tc::fma2(P[i + 2], P[i + 2], q2);
              q3 = tc::fma2(P[i + 3], P[i + 3], q3);
            }
            const float sc = sqrtf(__ldg(p.qk_scale + head)) * rsqrtf(((q0.x + q0.y) + (q1.x + q1.y)) + ((q2.x + q2.y) + (q3.x + q3.y)) + 1e-6f);
            const tc::f32x2 sc2 = tc::pk2(sc, sc);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 cs = __ldg(tb + (int64_t)i * p.T);
              const tc::f32x2 C = tc::pk2(cs.x, cs.y), S = tc::pk2(cs.z, cs.w);
              const tc::f32x2 X1 = P[i], X2 = P[8 + i];
              P[i] = tc::mul2(tc::fma2(X2, tc::neg2(S), tc::mul2(X1, C)), sc2);
              P[8 + i] = tc::mul2(tc::fma2(X1, S, tc::mul2(X2, C)), sc2);
            }
#pragma unroll
            for (int i = 16; i < 32; ++i) P[i] = tc::mul2(P[i], sc2);
#pragma unroll
            for (int i = 0; i < 32; ++i) tc::upk2(P[i], v[2 * i], v[2 * i + 1]);
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint4*>(cg + tc::sw128_offset(row, j)) =
              make_uint4(tc::pack_bf16x2(v[j * 8 + 0], v[j * 8 + 1]), tc::pack_bf16x2(v[j * 8 + 2], v[j * 8 + 3]),
                         tc::pack_bf16x2(v[j * 8 + 4], v[j * 8 + 5]), tc::pack_bf16x2(v[j * 8 + 6], v[j * 8 + 7]));
      }
    }
    if constexpr (RES || EPI == TCE_STORE) {
      if (p.ss_out != nullptr && m < p.M) p.ss_out[m * SS_PARTS + (n0 >> 7)] = (ss_acc[0] + ss_acc[1]) + (ss_acc[2] + ss_acc[3]);
    }
    tc::fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA (async proxy)
    tc::named_barrier_sync(1, 128);
    if (threadIdx.x == 0) {
      if constexpr (EPI == TCE_GEGLU) {
        tc::tma_store_2d(&tmc, sC, n0 / 2, (int)m0);
      } else {
#pragma unroll
        for (int g = 0; g < NSUB; ++g) tc::tma_store_2d(&tmc, sC + g * SUB_TILE_BYTES, n0 + g * 64, (int)m0);
      }
      tc::tma_store_commit();
      tc::tma_store_wait_read();             // smem must stay alive until the bulk store has read it
    }
  }
}

inline int num_sms() {
  static int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = kNumSMs;
    return v;
  }();
  return n;
}

#include "tc_ffn_fused.cuh"

// Ring depth: two CTAs stay co-resident per SM (one CTA's epilogue overlaps the other's main loop), so a 128-wide tile keeps two
// stages (the fp32 accumulator tile re-uses them) and a 64-wide tile up to four.
int pick_stages(int K, int BN) {
  const int nkb = K / BK, want = BN == 128 ? 2 : 4;
  return nkb < want ? (nkb < 1 ? 1 : nkb) : want;
}

template <int BN, int EPI>
int launch_tc(const bf16* A, const bf16* W, TcParams p, cudaStream_t st) {
  CUtensorMap ta, tb, tcm, tr;
  int rc;
  if (p.a_merge) {
    if ((rc = tmap_quad(&ta, A, p.mC, p.mwc, (uint64_t)p.M / p.mwc, p.box_w, p.box_h))) return rc;
  } else {
    if ((rc = tmap_2d(&ta, A, (uint64_t)p.K, (uint64_t)p.M, BK, BM))) return rc;
  }
  if ((rc = tmap_2d(&tb, W, (uint64_t)p.K, (uint64_t)p.N, BK, BN))) return rc;
  const uint64_t n_out = EPI == TCE_GEGLU ? (uint64_t)p.N / 2 : (uint64_t)p.N;
  if (EPI != TCE_SPLIT && EPI != TCE_PATCHOUT) {
    if ((rc = tmap_2d(&tcm, p.out, n_out, (uint64_t)p.M, 64, BM))) return rc;
  } else {
    tcm = ta;
  }
  if (EPI == TCE_RESID) {
    if ((rc = tmap_2d(&tr, p.resid, (uint64_t)p.N, (uint64_t)p.M, 64, BM))) return rc;
  } else {
    tr = ta;
  }
  p.stages = pick_stages(p.K, BN);
  const size_t smem = gemm_smem<BN, EPI>(p.stages);
  static bool attr_set = false;
  if (!attr_set) {
    KDB_CUDA(cudaFuncSetAttribute(gemm_wg_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem<BN, EPI>(MAX_STAGES)));
    attr_set = true;
  }
  dim3 grid((unsigned)(p.N / BN), (unsigned)ceil_div(p.M, BM));
  gemm_wg_kernel<BN, EPI><<<grid, GEMM_THREADS, smem, st>>>(ta, tb, tcm, tr, p);
  KDB_LAUNCH_CHECK(EPI == TCE_PATCHOUT ? F_PATCH_OUT : F_GEMM_TC, st);   // (the profiler's per-family bookkeeping only)
  return 0;
}

// 128-wide tiles whenever N allows: they emit the per-128-channel row statistics of the fused RMSNorm
template <int EPI>
int dispatch_bn(const bf16* A, const bf16* W, const TcParams& p, cudaStream_t st) {
  if (p.N % 128 == 0) return launch_tc<128, EPI>(A, W, p, st);
  return launch_tc<64, EPI>(A, W, p, st);
}

bool shape_ok(int64_t M, int N, int K) {
  return M > 0 && M < (65535LL * BM) && N >= 64 && N % 64 == 0 && K >= 64 && K % 64 == 0;
}

}  // namespace

namespace {
// ------------------------------------------------------------------------------------------------
// patch_in on the tensor core (reference image_transformer_v2.py:586-595,723-724): tokens = TokenMerge 4x4 of c_in * x, then
// Linear(48 -> C0).  The A tile [128 tokens x 64] is not a TMA box of the NCHW fp32 latent, so the warpgroup builds it: thread =
// token, 12 coalesced float4 loads (3 channels x 4 patch rows: consecutive tokens are consecutive 16-byte pieces of an image row),
// * c_in, bf16, six 16-byte swizzled shared-memory stores.  K is ordered (c, nh, nw) -- the weight copy made at finalize has its
// columns permuted to match and is zero-padded from 48 to 64.  One wgmma k-block, then the usual accumulator tile -> bf16 staging
// tile -> TMA store epilogue, which also leaves sum(x^2) per row for the fused RMSNorm.
// ------------------------------------------------------------------------------------------------
struct PatchInParams {
  const float* x;
  const float* sigma;
  float sd;
  int64_t M;
  int H, Wimg, th, tw, N;
  float* ss_out;
};

constexpr size_t PATCH_IN_SMEM = 1024 + 2 * A_STAGE_BYTES + (size_t)BM * acc_ld<128>() * 4 + 2 * SUB_TILE_BYTES + 64;

__global__ void __launch_bounds__(GEMM_THREADS) patch_in_tc_kernel(const __grid_constant__ CUtensorMap tmw, const __grid_constant__ CUtensorMap tmc,
                                                                   const PatchInParams p) {
  KDB_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  constexpr int LD = acc_ld<128>();
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = base;                       // [128 tokens x 64] bf16, SWIZZLE_128B
  uint8_t* sW = base + A_STAGE_BYTES;       // [128 outputs x 64]
  uint8_t* sC = sW + A_STAGE_BYTES;         // staging tile, two 64-column halves
  float* sAcc = reinterpret_cast<float*>(sC + 2 * SUB_TILE_BYTES);
  uint64_t* w_full = reinterpret_cast<uint64_t*>(sAcc + BM * LD);

  const int warp = threadIdx.x >> 5;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * 128;
  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmw);
    tc::tma_prefetch_desc(&tmc);
    tc::mbar_init(w_full, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (tc::elect_one()) {
      tc::mbar_arrive_expect_tx(w_full, A_STAGE_BYTES);
      tc::tma_load_2d(sW, &tmw, w_full, 0, n0);
    }
    return;
  }
  const int row = threadIdx.x;
  const int64_t m = m0 + row;
  // ---- gather: the token's 4x4x3 pixels
  uint4 chunk[6];
  if (m < p.M) {
    const int per = p.th * p.tw;
    const int b = (int)(m / per);
    const int r = (int)(m - (int64_t)b * per);
    const int ty = r / p.tw, tx = r - ty * p.tw;
    float c_in = 1.f;
    if (p.sd > 0.f) {
      const float sg = __ldg(p.sigma + b);
      c_in = rsqrtf(fmaf(sg, sg, p.sd * p.sd));
    }
    float4 px[12];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int nh = 0; nh < 4; ++nh)
        px[c * 4 + nh] = __ldg(reinterpret_cast<const float4*>(p.x + (((int64_t)b * 3 + c) * p.H + (ty * 4 + nh)) * p.Wimg + tx * 4));
#pragma unroll
    for (int j = 0; j < 6; ++j) {          // chunk j = K columns 8j .. 8j+7 = (c = j / 2, nh = 2 (j & 1) and 2 (j & 1) + 1)
      const float4 a = px[2 * j], bq = px[2 * j + 1];
      chunk[j] = make_uint4(tc::pack_bf16x2(a.x * c_in, a.y * c_in), tc::pack_bf16x2(a.z * c_in, a.w * c_in), tc::pack_bf16x2(bq.x * c_in, bq.y * c_in),
                            tc::pack_bf16x2(bq.z * c_in, bq.w * c_in));
    }
  } else {
#pragma unroll
    for (int j = 0; j < 6; ++j) chunk[j] = make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) *reinterpret_cast<uint4*>(sA + tc::sw128_offset(row, j)) = chunk[j];
  *reinterpret_cast<uint4*>(sA + tc::sw128_offset(row, 6)) = make_uint4(0u, 0u, 0u, 0u);     // K 48..63: zero padding
  *reinterpret_cast<uint4*>(sA + tc::sw128_offset(row, 7)) = make_uint4(0u, 0u, 0u, 0u);
  tc::fence_proxy_async();                 // generic-proxy writes -> visible to the tensor core's shared-memory reads
  tc::named_barrier_sync(1, 128);
  tc::mbar_wait(w_full, 0);
  {
    float acc0[64], acc1[64];
    const uint32_t a_addr = tc::smem_u32(sA);
    const uint64_t ad0 = tc::smem_desc_k_sw128(a_addr), ad1 = tc::smem_desc_k_sw128(a_addr + 8 * 1024), bd = tc::smem_desc_k_sw128(tc::smem_u32(sW));
#pragma unroll
    for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      tc::wgmma_128(acc0, ad0 + 2ull * k, bd + 2ull * k, 1u);
      tc::wgmma_128(acc1, ad1 + 2ull * k, bd + 2ull * k, 1u);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    tc::acc_store(sAcc, LD, 0, acc0);
    tc::acc_store(sAcc, LD, 64, acc1);
  }
  tc::named_barrier_sync(1, 128);
  // ---- epilogue
  float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    float v[64];
    {
      float t0[32], t1[32];
      tc::acc_ld32(sAcc, LD, row, g * 64, t0);
      tc::acc_ld32(sAcc, LD, row, g * 64 + 32, t1);
#pragma unroll
      for (int i = 0; i < 32; ++i) { v[i] = t0[i]; v[32 + i] = t1[i]; }
    }
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      ss0 = fmaf(v[i], v[i], ss0);
      ss1 = fmaf(v[i + 1], v[i + 1], ss1);
    }
    uint8_t* cg = sC + g * SUB_TILE_BYTES;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint4*>(cg + tc::sw128_offset(row, j)) =
          make_uint4(tc::pack_bf16x2(v[j * 8 + 0], v[j * 8 + 1]), tc::pack_bf16x2(v[j * 8 + 2], v[j * 8 + 3]),
                     tc::pack_bf16x2(v[j * 8 + 4], v[j * 8 + 5]), tc::pack_bf16x2(v[j * 8 + 6], v[j * 8 + 7]));
  }
  if (p.ss_out != nullptr && m < p.M) p.ss_out[m * SS_PARTS + (n0 >> 7)] = ss0 + ss1;
  tc::fence_proxy_async();
  tc::named_barrier_sync(1, 128);
  if (threadIdx.x == 0) {
    tc::tma_store_2d(&tmc, sC, n0, (int)m0);
    tc::tma_store_2d(&tmc, sC + SUB_TILE_BYTES, n0 + 64, (int)m0);
    tc::tma_store_commit();
    tc::tma_store_wait_read();
  }
}

// W [N, 48] fp32 with columns (nh, nw, c) -> bf16 [N, 64] with columns (c, nh, nw), zero-padded
__global__ void __launch_bounds__(256) patch_in_weight_kernel(const float* __restrict__ W, bf16* __restrict__ out, int N) {
  for (int i = blockIdx.x * 256 + threadIdx.x; i < N * 64; i += gridDim.x * 256) {
    const int n = i >> 6, k = i & 63;
    float v = 0.f;
    if (k < 48) {
      const int c = k >> 4, nh = (k >> 2) & 3, nw = k & 3;
      v = W[(int64_t)n * 48 + (nh * 4 + nw) * 3 + c];
    }
    out[i] = __float2bfloat16(v);
  }
}

}  // namespace

static bool g_tc_disabled = [] {
  const char* e = getenv("KDB200_DISABLE_TC");
  return e != nullptr && e[0] == '1';
}();

bool tc_gemm_supported(int64_t M, int N, int K, const GemmEpi& epi) {
  if (g_tc_disabled || !shape_ok(M, N, K)) return false;
  if (epi.ss_in != nullptr && (N % 128 != 0 || K % 128 != 0 || K > 128 * SS_PARTS || (epi.mode != EPI_STORE && epi.mode != EPI_QKV_ROPE) || epi.mC > 0))
    return false;
  if (epi.mC > 0) {   // TokenMerge gather folded into the A loads: 128-wide tiles, plain store epilogue
    int bw, bh;
    if (epi.mode != EPI_STORE || N % 128 != 0 || epi.mC % 64 != 0 || K != 4 * epi.mC || M % epi.mwc != 0 || !quad_box(epi.mwc, &bw, &bh)) return false;
  }
  if (epi.mode == EPI_SPLIT_LERP) return epi.C % 32 == 0 && N == 4 * epi.C;
  if (epi.mode == EPI_QKV_ROPE) return N == 3 * epi.C && epi.C % 64 == 0 && epi.nh * 64 == epi.C && epi.rope != nullptr;
  return epi.mode == EPI_STORE || epi.mode == EPI_RESID;
}

// true when the RESID / SPLIT / STORE GEMM of this shape runs on 128-wide tiles, which leave sum(x^2) of every row they write
bool tc_gemm_emits_rowss(int64_t M, int N, int K, const GemmEpi& epi) {
  if (!tc_gemm_supported(M, N, K, epi)) return false;
  if (N % 128 != 0) return false;
  if (epi.mode == EPI_RESID || epi.mode == EPI_STORE) return N <= 128 * SS_PARTS;   // (STORE: the TokenMerge projection)
  if (epi.mode == EPI_SPLIT_LERP) return epi.C % 128 == 0 && epi.C <= 128 * SS_PARTS;
  return false;
}

int launch_gemm_tc(const bf16* A, const bf16* W, bf16* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st) {
  KDB_REQUIRE(shape_ok(M, N, K), KDB_ERR_BAD_SHAPE, "gemm_tc: unsupported shape M=%lld N=%d K=%d", (long long)M, N, K);
  KDB_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0,
              KDB_ERR_BAD_ARG, "gemm_tc: operands must be 16-byte aligned");
  TcParams p{};
  p.out = C;
  p.M = M;
  p.N = N;
  p.K = K;
  p.ss_in = epi.ss_in;
  p.ss_out = epi.ss_out;
  KDB_REQUIRE(epi.ss_in == nullptr || tc_gemm_supported(M, N, K, epi), KDB_ERR_UNSUPPORTED, "gemm_tc: fused-norm geometry not supported");
  KDB_REQUIRE(epi.ss_out == nullptr || tc_gemm_emits_rowss(M, N, K, epi), KDB_ERR_UNSUPPORTED, "gemm_tc: this shape cannot emit row statistics");
  if (epi.mC > 0) {
    KDB_REQUIRE(tc_gemm_supported(M, N, K, epi), KDB_ERR_UNSUPPORTED, "gemm_tc: token-merge geometry not supported");
    p.a_merge = 1;
    p.mC = epi.mC;
    p.mwc = epi.mwc;
    quad_box(epi.mwc, &p.box_w, &p.box_h);
    return launch_tc<128, TCE_STORE>(A, W, p, st);
  }
  switch (epi.mode) {
    case EPI_STORE:
      return dispatch_bn<TCE_STORE>(A, W, p, st);
    case EPI_RESID:
      p.resid = static_cast<const bf16*>(epi.resid);
      return dispatch_bn<TCE_RESID>(A, W, p, st);
    case EPI_SPLIT_LERP:
      p.resid = static_cast<const bf16*>(epi.resid);
      p.fac = epi.fac;
      p.hc = epi.hc;
      p.wc = epi.wc;
      p.Cf = epi.C;
      return dispatch_bn<TCE_SPLIT>(A, W, p, st);
    case EPI_QKV_ROPE:
      p.rope = epi.rope;
      p.qk_scale = epi.qk_scale;
      p.C = epi.C;
      p.nh = epi.nh;
      p.T = epi.T_tokens;
      return dispatch_bn<TCE_QKV>(A, W, p, st);
    default:
      KDB_REQUIRE(false, KDB_ERR_BAD_ARG, "gemm_tc: bad epilogue");
  }
}

// patch_out on the tensor core: tokens already normalised (xn bf16 [M, C0]), W zero-padded to [64, C0]
bool tc_patch_out_supported(int C0, int Cout, int ph, int pw, int Wimg) {
  return !g_tc_disabled && C0 % 64 == 0 && Cout == 3 && ph == 4 && pw == 4 && Wimg % 4 == 0;
}

int launch_patch_out_tc(const bf16* xn, const bf16* W_pad, const float* x_in, const float* sigma, float sigma_data, float* out, int B, int H,
                        int Wimg, int C0, cudaStream_t st, const float* ss_in) {
  KDB_REQUIRE(ss_in == nullptr || (C0 % 128 == 0 && C0 <= 128 * SS_PARTS), KDB_ERR_UNSUPPORTED, "patch_out_tc: fused norm needs C0 %% 128 == 0");
  TcParams p{};
  p.ss_in = ss_in;
  p.M = (int64_t)B * (H / 4) * (Wimg / 4);
  p.N = 64;
  p.K = C0;
  p.fout = out;
  p.x_in = x_in;
  p.sigma = sigma;
  p.sd = sigma_data;
  p.H = H;
  p.Wimg = Wimg;
  p.th = H / 4;
  p.tw = Wimg / 4;
  KDB_REQUIRE(shape_ok(p.M, 64, C0), KDB_ERR_BAD_SHAPE, "patch_out_tc: unsupported shape");
  return launch_tc<64, TCE_PATCHOUT>(xn, W_pad, p, st);
}

bool tc_patch_in_supported(int Cin, int ph, int pw, int C0, int Wimg) {
  return !g_tc_disabled && Cin == 3 && ph == 4 && pw == 4 && C0 % 128 == 0 && C0 <= 128 * SS_PARTS && Wimg % 4 == 0;
}

int prepare_patch_in_weight(const float* W, bf16* out, int C0, cudaStream_t st) {
  patch_in_weight_kernel<<<(unsigned)ceil_div((int64_t)C0 * 64, 256), 256, 0, st>>>(W, out, C0);
  KDB_LAUNCH_CHECK(F_CONVERT, st);
  return 0;
}

int launch_patch_in_tc(const float* x, const float* sigma, float sigma_data, const bf16* W_perm, bf16* out, int B, int H, int Wimg, int C0,
                       float* ss_out, cudaStream_t st) {
  PatchInParams p{};
  p.x = x;
  p.sigma = sigma;
  p.sd = sigma_data;
  p.H = H;
  p.Wimg = Wimg;
  p.th = H / 4;
  p.tw = Wimg / 4;
  p.M = (int64_t)B * p.th * p.tw;
  p.N = C0;
  p.ss_out = ss_out;
  KDB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, KDB_ERR_BAD_ARG, "patch_in_tc: input must be 16-byte aligned");
  CUtensorMap tw, tcm;
  int rc;
  if ((rc = tmap_2d(&tw, W_perm, 64, (uint64_t)C0, 64, 128))) return rc;
  if ((rc = tmap_2d(&tcm, out, (uint64_t)C0, (uint64_t)p.M, 64, BM))) return rc;
  const size_t smem = PATCH_IN_SMEM;
  static bool attr_set = false;
  if (!attr_set) {
    KDB_CUDA(cudaFuncSetAttribute(patch_in_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  patch_in_tc_kernel<<<dim3((unsigned)ceil_div(p.M, BM), (unsigned)(C0 / 128)), GEMM_THREADS, smem, st>>>(tw, tcm, p);
  KDB_LAUNCH_CHECK(F_PATCH_IN, st);
  return 0;
}

bool tc_gemm_geglu_supported(int64_t M, int N2, int K, bool fused_norm) {
  if (fused_norm && (K % 128 != 0 || K > 128 * SS_PARTS)) return false;
  return !g_tc_disabled && shape_ok(M, N2, K) && N2 % 128 == 0;
}

__global__ void __launch_bounds__(256) fold_norm_weights_kernel(const FoldDesc* __restrict__ descs, const float* __restrict__ cond) {
  KDB_PDL_TRIGGER();
  const FoldDesc d = descs[blockIdx.y];
  const int64_t chunks = (int64_t)d.rows * d.K / 8;
  const float* g = cond + d.ada_off;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < chunks; i += (int64_t)gridDim.x * 256) {
    const int k0 = (int)((i * 8) % d.K);
    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(d.src) + i);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float lo = __uint_as_float(w[t] << 16) * __ldg(g + k0 + 2 * t), hi = __uint_as_float(w[t] & 0xffff0000u) * __ldg(g + k0 + 2 * t + 1);
      o[t] = tc::pack_bf16x2(lo, hi);
    }
    reinterpret_cast<uint4*>(d.dst)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int launch_fold_norm_weights(const FoldDesc* descs_dev, int n_desc, const float* cond_row, cudaStream_t st) {
  if (n_desc <= 0) return 0;
  fold_norm_weights_kernel<<<dim3(48, (unsigned)n_desc), 256, 0, st>>>(descs_dev, cond_row);
  KDB_LAUNCH_CHECK(F_FUSED_NORM, st);
  return 0;
}

int launch_gemm_tc_geglu(const bf16* A, const bf16* W_il, bf16* out, int64_t M, int N2, int K, cudaStream_t st, const float* ss_in) {
  KDB_REQUIRE(tc_gemm_geglu_supported(M, N2, K, ss_in != nullptr), KDB_ERR_BAD_SHAPE, "gemm_tc_geglu: unsupported shape");
  TcParams p{};
  p.ss_in = ss_in;
  p.out = out;
  p.M = M;
  p.N = N2;
  p.K = K;
  return launch_tc<128, TCE_GEGLU>(A, W_il, p, st);
}

bool tc_ffn_fused_supported(int64_t M, int C, int dff) {
  static const bool off = [] {
    const char* e = getenv("KDB200_NO_FFN_FUSE");
    return e != nullptr && e[0] == '1';
  }();
  return !off && !g_tc_disabled && ffn_fused_supported(M, C, dff);
}

int launch_ffn_fused(bf16* x, const bf16* w_up_il, const bf16* w_down, int64_t M, int C, int dff, const float* ss_in, float* ss_out, cudaStream_t st) {
  KDB_REQUIRE(ffn_fused_supported(M, C, dff) && ss_in != nullptr, KDB_ERR_BAD_SHAPE, "ffn_fused: unsupported shape (needs C = 128, M %% 128 == 0, d_ff %% 64 == 0)");
  return launch_ffn_fused_impl(x, w_up_il, w_down, M, dff, ss_in, ss_out, st);
}

}  // namespace kdb

extern "C" int kdb_gemm_bf16(const void* a, const void* w, void* c, int M, int N, int K, void* stream) {
  using namespace kdb;
  KDB_REQUIRE(a && w && c, KDB_ERR_BAD_ARG, "gemm_bf16: NULL operand");
  GemmEpi e;
  KDB_REQUIRE(shape_ok(M, N, K), KDB_ERR_UNSUPPORTED, "gemm_bf16: needs N %% 64 == 0 and K %% 64 == 0 (got M=%d N=%d K=%d)", M, N, K);
  return launch_gemm_tc(static_cast<const bf16*>(a), static_cast<const bf16*>(w), static_cast<bf16*>(c), M, N, K, e, (cudaStream_t)stream);
}

extern "C" int kdb_gemm_bf16_geglu(const void* a, const void* w_il, void* c, int M, int N2, int K, const float* ss_in, void* stream) {
  using namespace kdb;
  KDB_REQUIRE(a && w_il && c, KDB_ERR_BAD_ARG, "gemm_bf16_geglu: NULL operand");
  KDB_REQUIRE(tc_gemm_geglu_supported(M, N2, K, ss_in != nullptr), KDB_ERR_UNSUPPORTED,
              "gemm_bf16_geglu: needs N2 %% 128 == 0 and K %% 64 == 0 (K %% 128 == 0, K <= 1024 with ss_in); got M=%d N2=%d K=%d", M, N2, K);
  return launch_gemm_tc_geglu(static_cast<const bf16*>(a), static_cast<const bf16*>(w_il), static_cast<bf16*>(c), M, N2, K, (cudaStream_t)stream, ss_in);
}

extern "C" int kdb_ffn_fused_bf16(void* x, const void* w_up_il, const void* w_down, int M, int d_ff, const float* ss_in, float* ss_out, void* stream) {
  using namespace kdb;
  KDB_REQUIRE(x && w_up_il && w_down && ss_in, KDB_ERR_BAD_ARG, "ffn_fused_bf16: NULL operand");
  return launch_ffn_fused(static_cast<bf16*>(x), static_cast<const bf16*>(w_up_il), static_cast<const bf16*>(w_down), M, 128, d_ff, ss_in, ss_out,
                          (cudaStream_t)stream);
}
