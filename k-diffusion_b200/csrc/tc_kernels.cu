// tc_kernels.cu -- bf16 tensor-core GEMM for sm_90a: TMA (SWIZZLE_128B tiles) -> shared memory -> wgmma (fp32 accumulators in
// registers) -> fp32 shared-memory tile -> fused epilogue (thread = output row; GEGLU: on the accumulator fragments) -> swizzled
// shared tile -> TMA store (clipped at the M edge by the tensor map).
//
// C[M,N] = A[M,K] W[N,K]^T for every nn.Linear on the token stream (reference image_transformer_v2.py:126-139).
// Epilogues (GemmEpilogue): EPI_STORE; EPI_RESID, +residual (out_proj / down_proj, :396,:493; residual tile prefetched by TMA
// while the main loop runs); EPI_GEGLU (:89-95; rows of W interleaved 8 value / 8 gate); EPI_SPLIT_LERP, TokenSplit scatter + lerp
// (:618-621); EPI_QKV_ROPE, cosine-sim scaling + axial RoPE of q and k fused into the qkv projection (:106-114,187-199,245-248;
// cos/sin from a per-layer table); EPI_PATCH_OUT, TokenSplitWithoutSkip 4x4 to fp32 NCHW + the Karras combine (:598-607,:758-760).
// One descriptor (GemmEpi), one predicate (tc_gemm_supported) and one launcher (launch_gemm_tc) for all of them.
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

static int make_tmap(CUtensorMap* out, CUtensorMapDataType type, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
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
  CUresult r = fn(out, type, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  KDB_REQUIRE(r == CUDA_SUCCESS, KDB_ERR_BAD_ARG, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dim0 %llu, box0 %u)", (int)r,
              rank, (unsigned long long)dims[0], box[0]);
  return 0;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}

int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides_bytes, box);
}

int make_tmap_f16_sw64(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

int make_tmap_tokens(CUtensorMap* out, const void* base, uint64_t C, int B, int h, int w, uint32_t box_c, uint32_t box_w, uint32_t box_h) {
  const uint64_t dims[4] = {C, (uint64_t)w, (uint64_t)h, (uint64_t)B};
  const uint64_t strides[3] = {C * 2, C * 2 * w, C * 2 * w * h};
  const uint32_t box[4] = {box_c, box_w, box_h, 1};
  return make_tmap_bf16(out, base, 4, dims, strides, box);
}

// programmatic dependent launch for every kernel launched with launch_pdl, unless the switch below is 1 (read once, at the first launch)
bool pdl_enabled() {
  static const bool enabled = [] {
    const char* e = getenv("KDB200_NO_PDL");
    return !(e != nullptr && e[0] == '1');
  }();
  return enabled;
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int BM = 128, BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KiB
constexpr int SUB_TILE_BYTES = BM * 128;     // one [128 x 64] bf16 output sub-tile
constexpr int GEMM_THREADS = 384;            // warpgroups 0, 1: MMA + epilogue of alternate tiles, warpgroup 2: TMA producer (one warp)

// The kernel's parameter block: the epilogue descriptor, the output and the shape, and what launch_gemm_tc derives from them.
struct GemmArgs : GemmEpi {
  bf16* out;
  int64_t M;
  int N, K;
  int box_w, box_h;      // 5-D TMA box of the merge gather (mC > 0) or of the split scatter (EPI_SPLIT_LERP, box_w > 0): 128 rows =
                         // box_h x box_w coarse tokens
  int th, tw;            // EPI_PATCH_OUT: token grid H / 4 x W / 4
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

// TMA coordinates in tmap_quad's view of the [128 x 64] box that holds coarse rows m0.. (m0 % 128 == 0) and columns n.. of quadrant
// n / C: the same box for the merge's A loads (n = k, C = mC) and for the split's skip loads and output stores
struct QuadCoord {
  int e, nw, wx, nh, row;
};
__device__ __forceinline__ QuadCoord quad_coord(int64_t m0, int n, int C, int wc, int box_h) {
  const int qd = n / C;
  return QuadCoord{n - qd * C, qd & 1, box_h == 1 ? (int)(m0 % wc) : 0, qd >> 1, (int)(m0 / wc)};
}

// Shared memory of one GEMM CTA: the TMA ring, the fp32 accumulator tile (shared by the two warpgroups, in tile order), per
// warpgroup the bf16 output staging tile (RESID: the residual tile is loaded into it and the epilogue adds in place), then the
// barriers.  The fp32 tile holds 64 columns of the 128 x BN accumulators at a time (a 128-wide epilogue stages its second half once
// every thread has read the first), so 128-wide RESID / STORE / QKV / SPLIT take 128 + 32 + 2 x 32 KiB + 1 KiB of alignment = 225 KiB:
// 4 ring stages instead of the 3 a whole 64 KiB fp32 tile leaves room for.  GEGLU runs its epilogue on the accumulator fragments and
// has no fp32 tile: 6 stages of 32 KiB + 2 x 16 KiB + 1 KiB = 225 KiB.
template <int BN, int EPI> constexpr int out_bytes() {
  return EPI == EPI_GEGLU ? SUB_TILE_BYTES : EPI == EPI_PATCH_OUT ? 0 : (BN / 64) * SUB_TILE_BYTES;
}
constexpr int ACC_COLS = 64;                 // columns of the fp32 accumulator tile
template <int BN, int EPI> constexpr int acc_bytes() { return EPI == EPI_GEGLU ? 0 : BM * ACC_COLS * 4; }
template <int EPI> constexpr int ring_bytes() { return EPI == EPI_GEGLU ? 192 * 1024 : 128 * 1024; }   // 128 KiB: 4 stages of 128-wide tiles, 5 of 64-wide
template <int BN, int EPI> constexpr size_t gemm_smem() { return 1024 + ring_bytes<EPI>() + acc_bytes<BN, EPI>() + 2 * out_bytes<BN, EPI>() + 128; }

// The fp32 accumulator tile is [128 rows x 64 columns] with the 16-byte chunks of row r XOR-swizzled by r % 8: the fragment stores
// (8 rows x 4 column pairs per warp) and the row reads (32 rows, one float4 each) both spread evenly over the banks.
__device__ __forceinline__ int stage_off(int row, int chunk) { return row * ACC_COLS + ((chunk ^ (row & 7)) << 2); }
// columns [64 H, 64 H + 64) of the accumulator fragment of rows [row0, row0 + 64) -> the fp32 tile
template <int BN, int H>
__device__ __forceinline__ void stage_store(float* s, int row0, const float (&d)[BN / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < ACC_COLS / 8; ++j) {
    const int jd = H * (ACC_COLS / 8) + j;   // 8-column block of the fragment
    *reinterpret_cast<float2*>(s + stage_off(r, 2 * j + (c >> 2)) + (c & 3)) = make_float2(d[4 * jd], d[4 * jd + 1]);
    *reinterpret_cast<float2*>(s + stage_off(r + 8, 2 * j + (c >> 2)) + (c & 3)) = make_float2(d[4 * jd + 2], d[4 * jd + 3]);
  }
}
// Columns 64..127 of a 128-wide tile replace columns 0..63 in the fp32 tile, once every thread of the warpgroup has read those
template <int BN>
__device__ __forceinline__ void stage_second_half(float* s, int wg, const float (&acc0)[BN / 2], const float (&acc1)[BN / 2]) {
  if constexpr (BN == 128) {
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
    stage_store<BN, 1>(s, 0, acc0);
    stage_store<BN, 1>(s, 64, acc1);
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
  }
}
// 32 consecutive columns of one row of the fp32 tile; col0 is the column in the 128 x BN tile (the half it lies in is staged)
__device__ __forceinline__ void stage_ld32(const float* s, int row, int col0, float (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 q = *reinterpret_cast<const float4*>(s + stage_off(row, ((col0 % ACC_COLS) >> 2) + i));
    v[4 * i] = q.x;
    v[4 * i + 1] = q.y;
    v[4 * i + 2] = q.z;
    v[4 * i + 3] = q.w;
  }
}
__device__ __forceinline__ void stage_ld64(const float* s, int row, int col0, float (&v)[64]) {
  float t0[32], t1[32];
  stage_ld32(s, row, col0, t0);
  stage_ld32(s, row, col0 + 32, t1);
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    v[k] = t0[k];
    v[32 + k] = t1[k];
  }
}

// C[M,N] in 128 x BN tiles, N-fastest inside a 128-row block so that the CTAs at work share A in L2; CTA b takes tiles b, b + grid,
// b + 2 grid, ... and its warpgroup w the odd / even ones of those.  Warp 8 (one elected lane) streams the A / W k-blocks of the
// CTA's tiles, in tile order, through one ring of SWIZZLE_128B stages, so the next tile's k-blocks load during an epilogue.  A
// warpgroup issues wgmma (two M = 64 halves per k-step) with the accumulators in registers, keeps one k-block in flight while it
// releases the previous stage, and hands the MMA issue to the other warpgroup once its last k-block is issued (BAR_TURN: the two
// main loops never interleave, which also keeps each ring stage at most one phase ahead of its waiter).  Its epilogue then
// writes the accumulators to the fp32 tile in shared memory so that each thread owns one output row (fp32 arithmetic, one rounding
// to bf16 at the pack, one TMA store per 64 columns), and hands the fp32 tile on once its rows are read (BAR_ACC).  GEGLU works
// element by element on value / gate pairs that share a thread: it runs on the accumulator fragments themselves and writes bf16
// pairs straight into its staging tile, without the fp32 tile or BAR_ACC.
// ROPE_R: EPI_QKV_ROPE's rotated width R when it is not 32 (one value: image_transformer_v1 rotates all 64 columns of a head); the
// other instantiations keep an empty pack, and with it their demangled names (gemm_wg_kernel<64, 5>, which profilers report).
template <int... R> struct RopeWidth { static constexpr int value = 32; };
template <int R> struct RopeWidth<R> { static constexpr int value = R; };

template <int BN, int EPI, int... ROPE_R>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wg_kernel(const __grid_constant__ CUtensorMap tma, const __grid_constant__ CUtensorMap tmb,
                                                                  const __grid_constant__ CUtensorMap tmc, const __grid_constant__ CUtensorMap tmr,
                                                                  const GemmArgs p) {
  KDB_PDL_TRIGGER();
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  constexpr int RING_BYTES = ring_bytes<EPI>();
  constexpr int STAGES = RING_BYTES / STAGE_BYTES;
  constexpr int NSUB = BN / 64;
  constexpr bool RES = EPI == EPI_RESID;
  uint8_t* base = tc::smem_1k();
  float* sAcc = reinterpret_cast<float*>(base + RING_BYTES);
  auto* ring = reinterpret_cast<tc::TmaRing<STAGES>*>(base + RING_BYTES + acc_bytes<BN, EPI>() + 2 * out_bytes<BN, EPI>());
  uint64_t* resid_full = reinterpret_cast<uint64_t*>(ring + 1);   // one per warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = p.K / BK;
  const int n_tiles = p.N / BN;
  const int n_local = tc::tiles_owned((int)((p.M + BM - 1) / BM) * n_tiles);

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tma);
    tc::tma_prefetch_desc(&tmb);
    ring->init(tc::REL_WARPS);           // by the warpgroup that consumes the k-block
    tc::mbar_init(&resid_full[0], 1);
    tc::mbar_init(&resid_full[1], 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::pdl_wait();   // A, the residual, the row statistics and W (folded for this evaluation) are written by the kernels before us

  if (warp >= 8) {
    tc::setmaxnreg_dec<tc::PRODUCER_REGS>();
    if (warp == 8 && tc::elect_one()) {
      int it = 0;                        // ring position of the next k-block
      for (int i = 0; i < n_local; ++i) {
        const int t = (int)blockIdx.x + i * (int)gridDim.x;
        const int64_t m0 = (int64_t)(t / n_tiles) * BM;
        const int n0 = (t % n_tiles) * BN;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const auto ps = PipeState<STAGES>::at(it);
          uint64_t* bar = ring->acquire(ps, STAGE_BYTES);
          uint8_t* a = base + (size_t)ps.slot * STAGE_BYTES;
          if (p.mC > 0) {    // TokenMerge: k-block kb lives in quadrant (nh, nw) of the fine grid, channels e0..e0+63
            const QuadCoord q = quad_coord(m0, kb * BK, p.mC, p.mwc, p.box_h);
            tc::tma_load_5d(a, &tma, bar, q.e, q.nw, q.wx, q.nh, q.row);
          } else {
            tc::tma_load_2d(a, &tma, bar, kb * BK, (int)m0);
          }
          tc::tma_load_2d(a + A_STAGE_BYTES, &tmb, bar, kb * BK, n0);
        }
      }
    }
    return;
  }
  tc::setmaxnreg_inc<tc::MMA_REGS>();

  const int wg = warp >> 2;
  const int row = threadIdx.x & 127;
  uint8_t* sC = base + RING_BYTES + acc_bytes<BN, EPI>() + wg * out_bytes<BN, EPI>();
  const int r0 = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);   // fragment rows r0, r0 + 8 (+ 64 in acc1), column pair cq
  for (int i = wg; i < n_local; i += 2) {
    const int t = (int)blockIdx.x + i * (int)gridDim.x;
    const int64_t m0 = (int64_t)(t / n_tiles) * BM;
    const int n0 = (t % n_tiles) * BN;
    // the residual / skip tile by TMA into sC; the previous tile's store has finished reading sC (tma_store_wait_read below)
    if constexpr (RES || EPI == EPI_SPLIT_LERP) {
      if (row == 0 && (RES || p.box_w > 0)) {
        tc::mbar_arrive_expect_tx(&resid_full[wg], NSUB * SUB_TILE_BYTES);
#pragma unroll
        for (int g = 0; g < NSUB; ++g) {
          if constexpr (RES) {
            tc::tma_load_2d(sC + g * SUB_TILE_BYTES, &tmr, &resid_full[wg], n0 + g * 64, (int)m0);
          } else {
            const QuadCoord q = quad_coord(m0, n0 + g * 64, p.C, p.wc, p.box_h);
            tc::tma_load_5d(sC + g * SUB_TILE_BYTES, &tmr, &resid_full[wg], q.e, q.nw, q.wx, q.nh, q.row);
          }
        }
      }
    }
    // GEGLU: 1/rms of the fragment rows r0, r0 + 8, 64 + r0, 72 + r0, loaded while the other warpgroup's main loop runs
    float frag_rstd[4] = {1.f, 1.f, 1.f, 1.f};
    if constexpr (EPI == EPI_GEGLU) {
      if (p.ss_in != nullptr) {
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int64_t m = m0 + r0 + 64 * (h >> 1) + 8 * (h & 1);
          const float4* sp = reinterpret_cast<const float4*>(p.ss_in + (m < p.M ? m : 0) * SS_PARTS);
          frag_rstd[h] = rsqrtf(tc::rowss_sum(__ldg(sp), __ldg(sp + 1), p.K >> 7) / (float)p.K + 1e-6f);
        }
      }
    }

    // ---------------- main loop: warpgroup MMA, accumulators in registers
    float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
    for (int k = 0; k < BN / 2; ++k) acc0[k] = acc1[k] = 0.f;
    if (i > 0) tc::named_barrier_sync(tc::BAR_TURN + wg, 256);   // the other warpgroup has issued the main loop of tile i - 1
    const int it0 = i * nkb;             // ring position of this tile's first k-block
    for (int kb = 0; kb < nkb; ++kb) {
      const auto ps = PipeState<STAGES>::at(it0 + kb);
      ring->wait(ps);
      const uint32_t a_addr = tc::smem_u32(base + (size_t)ps.slot * STAGE_BYTES);
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
      if (kb > 0 && lane == 0) ring->release(PipeState<STAGES>::at(it0 + kb - 1));
    }
    if (i + 1 < n_local) tc::named_barrier_arrive(tc::BAR_TURN + (wg ^ 1), 256);
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc0);
    tc::wg_fence_acc(acc1);
    if (lane == 0) ring->release(PipeState<STAGES>::at(it0 + nkb - 1));

    if constexpr (EPI == EPI_GEGLU) {
      // ---------------- epilogue on the fragments: output column 8q + cq of row r = GEGLU of the pair in 8-column blocks 2q, 2q + 1
      tc::named_barrier_sync(tc::BAR_WG + wg, 128);   // row 0 has seen the previous tile's store finish reading sC
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const float r_a = frag_rstd[2 * half], r_b = frag_rstd[2 * half + 1];
        uint32_t o[16];
        tc::geglu_fragment(half == 0 ? acc0 : acc1, tc::pk2(0.5f * r_a, 0.5f * r_a), tc::pk2(0.5f * r_b, 0.5f * r_b), tc::pk2(r_a, r_a),
                           tc::pk2(r_b, r_b), o);
        const int r = 64 * half + r0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          *reinterpret_cast<uint32_t*>(sC + tc::sw128_offset(r, q) + 2 * cq) = o[2 * q];
          *reinterpret_cast<uint32_t*>(sC + tc::sw128_offset(r + 8, q) + 2 * cq) = o[2 * q + 1];
        }
      }
      tc::fence_proxy_async();
      tc::named_barrier_sync(tc::BAR_WG + wg, 128);
      if (row == 0) {
        tc::tma_store_2d(&tmc, sC, n0 / 2, (int)m0);
        tc::tma_store_commit();
        tc::tma_store_wait_read();
      }
      continue;
    }
    if (i > 0) tc::named_barrier_sync(tc::BAR_ACC + wg, 256);   // the other warpgroup has read tile i - 1 out of the fp32 tile
    stage_store<BN, 0>(sAcc, 0, acc0);
    stage_store<BN, 0>(sAcc, 64, acc1);
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
    const bool pass_acc = i + 1 < n_local;   // after its last read of the fp32 tile this warpgroup hands it on (named_barrier_arrive)

    // ---------------- epilogue: thread = output row
    const int64_t m = m0 + row;
    float rstd = 1.f;
    if (p.ss_in != nullptr) {   // fused RMSNorm (consumer side): the producer of x left sum(x^2) of every token, one slot per 128 channels
      const float4* sp = reinterpret_cast<const float4*>(p.ss_in + (m < p.M ? m : 0) * SS_PARTS);
      rstd = rsqrtf(tc::rowss_sum(__ldg(sp), __ldg(sp + 1), p.K >> 7) / (float)p.K + 1e-6f);
    }
    if constexpr (EPI == EPI_PATCH_OUT) {
      // TokenSplitWithoutSkip 4x4 + NCHW + Denoiser combine (reference :598-607,:758-760, layers.py:88-90).  Row m = token
      // (b, ty, tx); column n = (nh*4 + nw)*3 + c.  For fixed (c, nh) the 4 nw pixels are one float4.
      float v[64];
      {
        float t0[32], t1[32];
        stage_ld32(sAcc, row, 0, t0);
        stage_ld32(sAcc, row, 32, t1);
#pragma unroll
        for (int k = 0; k < 32; ++k) { v[k] = t0[k]; v[32 + k] = t1[k]; }
      }
      if (pass_acc) tc::named_barrier_arrive(tc::BAR_ACC + (wg ^ 1), 256);
      if (m < p.M) {
        if (p.ss_in != nullptr) {   // fused out_norm: A is the raw residual stream, W carries the channel scale
#pragma unroll
          for (int k = 0; k < 48; ++k) v[k] *= rstd;
        }
        const int per = p.th * p.tw;
        const int b = (int)(m / per);
        const int r = (int)(m - (int64_t)b * per);
        const int ty = r / p.tw, tx = r - ty * p.tw;
        float c_skip = 0.f, c_out = 1.f, c_in;
        if (p.sigma_data > 0.f) karras_scalings(__ldg(p.sigma + b), p.sigma_data, c_skip, c_out, c_in);
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int nh = 0; nh < 4; ++nh) {
            const int64_t o = (((int64_t)b * 3 + c) * p.H + (ty * 4 + nh)) * p.W + tx * 4;
            float4 y = make_float4(bf16_round(v[(nh * 4 + 0) * 3 + c]), bf16_round(v[(nh * 4 + 1) * 3 + c]), bf16_round(v[(nh * 4 + 2) * 3 + c]),
                                   bf16_round(v[(nh * 4 + 3) * 3 + c]));
            if (p.sigma_data > 0.f) {
              const float4 xi = __ldg(reinterpret_cast<const float4*>(p.x_in + o));
              y = make_float4(y.x * c_out + xi.x * c_skip, y.y * c_out + xi.y * c_skip, y.z * c_out + xi.z * c_skip, y.w * c_out + xi.w * c_skip);
            }
            *reinterpret_cast<float4*>(p.img + o) = y;
          }
      }
    } else if constexpr (EPI == EPI_SPLIT_LERP) {
      // TokenSplit + torch.lerp(skip, x, fac) (reference :618-621): row m = (b, hy, wx) on the coarse grid, column n = (quadrant
      // (nh, nw), channel e), scattered to the fine token, the lerp torch's (lerp_torch); sum(x^2) runs in column order.
      const bool live = m < p.M;
      const float facv = __ldg(p.fac);
      float ss = 0.f;
      int64_t fine = 0;
      if (p.box_w > 0) {
        // 64 columns of one quadrant x 128 coarse rows are one box of the quadrant maps: the skip tile arrived by TMA under the main
        // loop, the lerp runs in place (each thread its own row), and the tile leaves by TMA store through the same box of `out`
        tc::mbar_wait_nocall(&resid_full[wg], (uint32_t)(i >> 1) & 1u);
#pragma unroll 1
        for (int g = 0; g < NSUB; ++g) {
          if (g == 1) stage_second_half<BN>(sAcc, wg, acc0, acc1);
          float v[64];
          {
            float t0[32], t1[32];
            stage_ld32(sAcc, row, g * 64, t0);
            stage_ld32(sAcc, row, g * 64 + 32, t1);
#pragma unroll
            for (int k = 0; k < 32; ++k) { v[k] = t0[k]; v[32 + k] = t1[k]; }
          }
          if (g == NSUB - 1 && pass_acc) tc::named_barrier_arrive(tc::BAR_ACC + (wg ^ 1), 256);
          uint8_t* cg = sC + g * SUB_TILE_BYTES;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            uint4* cp = reinterpret_cast<uint4*>(cg + tc::sw128_offset(row, j));
            const uint4 r4 = *cp;
            const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
            uint32_t ow[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float lo = __uint_as_float(rw[q] << 16), hi = __uint_as_float(rw[q] & 0xffff0000u);
              const float e0 = v[j * 8 + q * 2], e1 = v[j * 8 + q * 2 + 1];
              const float o0 = lerp_torch(lo, e0, facv);
              const float o1 = lerp_torch(hi, e1, facv);
              ss = fmaf(o0, o0, fmaf(o1, o1, ss));
              ow[q] = tc::pack_bf16x2(o0, o1);
            }
            *cp = make_uint4(ow[0], ow[1], ow[2], ow[3]);
          }
        }
        if (p.ss_out != nullptr && live) {
          const int64_t b = m / ((int64_t)p.hc * p.wc);
          const int r = (int)(m - b * p.hc * p.wc);
          const int hy = r / p.wc, wx = r - hy * p.wc, qd = n0 / p.C;
          fine = (b * (2 * p.hc) + (2 * hy + (qd >> 1))) * (2 * p.wc) + (2 * wx + (qd & 1));
          p.ss_out[fine * SS_PARTS + ((n0 % p.C) >> 7)] = ss;
        }
        tc::fence_proxy_async();
        tc::named_barrier_sync(tc::BAR_WG + wg, 128);
        if (row == 0) {
#pragma unroll
          for (int g = 0; g < NSUB; ++g) {
            const QuadCoord q = quad_coord(m0, n0 + g * 64, p.C, p.wc, p.box_h);
            tc::tma_store_5d(&tmc, sC + g * SUB_TILE_BYTES, q.e, q.nw, q.wx, q.nh, q.row);
          }
          tc::tma_store_commit();
          tc::tma_store_wait_read();
        }
        continue;
      }
      // Coarse grids whose 128-row blocks are no box of the quadrant map (quad_box fails: wc >= 128 and not a multiple of 128, or
      // wc < 128 and not a divisor of it) and C % 64 != 0: 32 columns inside one quadrant (C % 32 == 0) per step, per-thread global
      // loads of the skip and stores of the output
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        if (c == 2) stage_second_half<BN>(sAcc, wg, acc0, acc1);
        float v[32];
        stage_ld32(sAcc, row, c * 32, v);
        if (c == BN / 32 - 1 && pass_acc) tc::named_barrier_arrive(tc::BAR_ACC + (wg ^ 1), 256);
        if (!live) continue;
        const int n = n0 + c * 32;
        const int64_t b = m / ((int64_t)p.hc * p.wc);
        const int r = (int)(m - b * p.hc * p.wc);
        const int hy = r / p.wc, wx = r - hy * p.wc;
        const int qd = n / p.C, e = n - qd * p.C;
        fine = (b * (2 * p.hc) + (2 * hy + (qd >> 1))) * (2 * p.wc) + (2 * wx + (qd & 1));
        const int64_t off = fine * p.C + e;
        const uint4* sk = reinterpret_cast<const uint4*>(static_cast<const bf16*>(p.resid) + off);
        uint4* dst = reinterpret_cast<uint4*>(p.out + off);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 r4 = sk[j];
          const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
          uint32_t ow[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float lo = __uint_as_float(rw[q] << 16), hi = __uint_as_float(rw[q] & 0xffff0000u);   // bf16 -> fp32 is a shift / mask
            const float e0 = v[j * 8 + q * 2], e1 = v[j * 8 + q * 2 + 1];
            const float o0 = lerp_torch(lo, e0, facv);
            const float o1 = lerp_torch(hi, e1, facv);
            ss = fmaf(o0, o0, fmaf(o1, o1, ss));
            ow[q] = tc::pack_bf16x2(o0, o1);
          }
          dst[j] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
      }
      // statistics of the new residual stream for the next fused RMSNorm (BN = 128 inside one quadrant: C % 128 == 0)
      if (p.ss_out != nullptr && live) p.ss_out[fine * SS_PARTS + ((n0 % p.C) >> 7)] = ss;
    } else {
      if constexpr (RES) tc::mbar_wait_nocall(&resid_full[wg], (uint32_t)(i >> 1) & 1u);
      float ss_acc[4] = {0.f, 0.f, 0.f, 0.f};   // producer side: sum of squares of the row this thread writes
      float v[64];
      stage_ld64(sAcc, row, 0, v);
      stage_second_half<BN>(sAcc, wg, acc0, acc1);   // the fragments are dead from here on
#pragma unroll 1
      for (int g = 0; g < NSUB; ++g) {
        if (g > 0) stage_ld64(sAcc, row, g * 64, v);
        if (g == NSUB - 1 && pass_acc) tc::named_barrier_arrive(tc::BAR_ACC + (wg ^ 1), 256);
        if (p.ss_in != nullptr) {
          // fused RMSNorm row scale.  q and k are cosine-normalised afterwards (scale invariant): only v needs it.
          bool apply = true;
          if constexpr (EPI == EPI_QKV_ROPE) apply = (n0 + g * 64) >= 2 * p.C;
          if (apply) {
#pragma unroll
            for (int k = 0; k < 64; ++k) v[k] *= rstd;
          }
        }
        uint8_t* cg = sC + g * SUB_TILE_BYTES;
        if constexpr (RES) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {      // this thread reads and then overwrites only its own row
            const uint4 r4 = *reinterpret_cast<const uint4*>(cg + tc::sw128_offset(row, j));
            const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              v[j * 8 + q * 2] += __uint_as_float(rw[q] << 16);
              v[j * 8 + q * 2 + 1] += __uint_as_float(rw[q] & 0xffff0000u);
            }
          }
        }
        if constexpr (RES || EPI == EPI_STORE) {
          if (p.ss_out != nullptr) {
#pragma unroll
            for (int k = 0; k < 64; k += 4) {
              ss_acc[0] = fmaf(v[k], v[k], ss_acc[0]);
              ss_acc[1] = fmaf(v[k + 1], v[k + 1], ss_acc[1]);
              ss_acc[2] = fmaf(v[k + 2], v[k + 2], ss_acc[2]);
              ss_acc[3] = fmaf(v[k + 3], v[k + 3], ss_acc[3]);
            }
          }
        }
        if constexpr (EPI == EPI_QKV_ROPE) {
          const int n = n0 + g * 64;               // one head of q, k or v (feature order (t nh e), d_head 64)
          const int t3 = n / p.C, head = (n - t3 * p.C) >> 6;
          if (t3 < 2) {
            // cosine-sim scale + axial RoPE (reference :106-114,187-199,245-248; QkRope).  Columns (2i, 2i+1) pair with (R/2+2i,
            // R/2+1+2i); the table holds (cos_2i, cos_2i+1, sin_2i, sin_2i+1) per float4, R/4 of them per head.
            constexpr int RQ = RopeWidth<ROPE_R...>::value / 4;
            static_assert(RQ * 4 <= 64 && RQ % 4 == 0, "rotated width must be a multiple of 16, at most d_head 64");
            const int64_t tok = (m < p.M ? m : 0) % p.T_tokens;
            const float4* tb = reinterpret_cast<const float4*>(p.rope) + (int64_t)head * RQ * p.T_tokens + tok;   // [head][i][token]
            tc::f32x2 P[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) P[k] = tc::pk2(v[2 * k], v[2 * k + 1]);
            tc::f32x2 q0 = tc::mul2(P[0], P[0]), q1 = tc::mul2(P[1], P[1]), q2 = tc::mul2(P[2], P[2]), q3 = tc::mul2(P[3], P[3]);
#pragma unroll
            for (int k = 4; k < 32; k += 4) {
              q0 = tc::fma2(P[k], P[k], q0);
              q1 = tc::fma2(P[k + 1], P[k + 1], q1);
              q2 = tc::fma2(P[k + 2], P[k + 2], q2);
              q3 = tc::fma2(P[k + 3], P[k + 3], q3);
            }
            const float sc = sqrtf(__ldg(p.qk_scale + head)) * rsqrtf(((q0.x + q0.y) + (q1.x + q1.y)) + ((q2.x + q2.y) + (q3.x + q3.y)) + p.qk_eps);
            const tc::f32x2 sc2 = tc::pk2(sc, sc);
#pragma unroll
            for (int k = 0; k < RQ; ++k) {
              const float4 cs = __ldg(tb + (int64_t)k * p.T_tokens);
              const tc::f32x2 C = tc::pk2(cs.x, cs.y), S = tc::pk2(cs.z, cs.w);
              const tc::f32x2 X1 = P[k], X2 = P[RQ + k];
              P[k] = tc::mul2(tc::fma2(X2, tc::neg2(S), tc::mul2(X1, C)), sc2);
              P[RQ + k] = tc::mul2(tc::fma2(X1, S, tc::mul2(X2, C)), sc2);
            }
#pragma unroll
            for (int k = 2 * RQ; k < 32; ++k) P[k] = tc::mul2(P[k], sc2);
#pragma unroll
            for (int k = 0; k < 32; ++k) tc::upk2(P[k], v[2 * k], v[2 * k + 1]);
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint4*>(cg + tc::sw128_offset(row, j)) =
              make_uint4(tc::pack_bf16x2(v[j * 8 + 0], v[j * 8 + 1]), tc::pack_bf16x2(v[j * 8 + 2], v[j * 8 + 3]),
                         tc::pack_bf16x2(v[j * 8 + 4], v[j * 8 + 5]), tc::pack_bf16x2(v[j * 8 + 6], v[j * 8 + 7]));
      }
      if constexpr (RES || EPI == EPI_STORE) {
        if (p.ss_out != nullptr && m < p.M) p.ss_out[m * SS_PARTS + (n0 >> 7)] = (ss_acc[0] + ss_acc[1]) + (ss_acc[2] + ss_acc[3]);
      }
      tc::fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA (async proxy)
      tc::named_barrier_sync(tc::BAR_WG + wg, 128);
      if (row == 0) {
#pragma unroll
        for (int g = 0; g < NSUB; ++g) tc::tma_store_2d(&tmc, sC + g * SUB_TILE_BYTES, n0 + g * 64, (int)m0);
        tc::tma_store_commit();
        tc::tma_store_wait_read();             // sC stays alive until the bulk store has read it; the next tile re-fills it
      }
    }
  }
}


#include "tc_ffn_fused.cuh"
#include "tc_attn_block.cuh"

template <int BN, int EPI, int... ROPE_R>
int launch_tc(const bf16* A, const bf16* W, const GemmArgs& p, cudaStream_t st) {
  CUtensorMap ta, tb, tcm, tr;
  int rc;
  if (p.mC > 0) {
    if ((rc = tmap_quad(&ta, A, p.mC, p.mwc, (uint64_t)p.M / p.mwc, p.box_w, p.box_h))) return rc;
  } else {
    if ((rc = tmap_2d(&ta, A, (uint64_t)p.K, (uint64_t)p.M, BK, BM))) return rc;
  }
  if ((rc = tmap_2d(&tb, W, (uint64_t)p.K, (uint64_t)p.N, BK, BN))) return rc;
  const uint64_t n_out = EPI == EPI_GEGLU ? (uint64_t)p.N / 2 : (uint64_t)p.N;
  if (EPI == EPI_SPLIT_LERP && p.box_w > 0) {   // skip and out: fine token tensors [B, 2 hc, 2 wc, C] in quadrant view
    if ((rc = tmap_quad(&tcm, p.out, p.C, p.wc, (uint64_t)p.M / p.wc, p.box_w, p.box_h))) return rc;
    if ((rc = tmap_quad(&tr, p.resid, p.C, p.wc, (uint64_t)p.M / p.wc, p.box_w, p.box_h))) return rc;
  } else {
    if (EPI != EPI_SPLIT_LERP && EPI != EPI_PATCH_OUT) {
      if ((rc = tmap_2d(&tcm, p.out, n_out, (uint64_t)p.M, 64, BM))) return rc;
    } else {
      tcm = ta;
    }
    if (EPI == EPI_RESID) {
      if ((rc = tmap_2d(&tr, p.resid, (uint64_t)p.N, (uint64_t)p.M, 64, BM))) return rc;
    } else {
      tr = ta;
    }
  }
  constexpr size_t smem = gemm_smem<BN, EPI>();
  static_assert(smem <= 227 * 1024, "GEMM shared memory exceeds the 227 KiB opt-in limit");
  static bool opened = false;
  if ((rc = set_smem_once(gemm_wg_kernel<BN, EPI, ROPE_R...>, opened, (int)smem))) return rc;
  KDB_CUDA(launch_pdl(gemm_wg_kernel<BN, EPI, ROPE_R...>, persistent_grid(ceil_div(p.M, BM) * (p.N / BN)), dim3(GEMM_THREADS), smem, st, ta, tb, tcm, tr, p));
  KDB_LAUNCH_CHECK(EPI == EPI_PATCH_OUT ? F_PATCH_OUT : F_GEMM_TC, st);   // (the profiler's per-family bookkeeping only)
  return 0;
}

// 128-wide tiles whenever N allows: they emit the per-128-channel row statistics of the fused RMSNorm
template <int EPI, int... ROPE_R>
int dispatch_bn(const bf16* A, const bf16* W, const GemmArgs& p, cudaStream_t st) {
  if (p.N % 128 == 0) return launch_tc<128, EPI, ROPE_R...>(A, W, p, st);
  return launch_tc<64, EPI, ROPE_R...>(A, W, p, st);
}

bool shape_ok(int64_t M, int N, int K) {
  return M > 0 && M < (65535LL * BM) && N >= 64 && N % 64 == 0 && K >= 64 && K % 64 == 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// the epilogue of this mode and N writes one row-statistics slot per 128 output channels (128-wide tiles, at most SS_PARTS slots)
bool rowss_fits(int N, const GemmEpi& epi) {
  if (N % 128 != 0) return false;
  if (epi.mode == EPI_RESID || epi.mode == EPI_STORE) return N <= 128 * SS_PARTS;   // (STORE: the TokenMerge projection)
  if (epi.mode == EPI_SPLIT_LERP) return epi.C % 128 == 0 && epi.C <= 128 * SS_PARTS;
  return false;
}

// Everything gemm_wg_kernel needs of the problem and its epilogue.
bool gemm_fits(int64_t M, int N, int K, const GemmEpi& epi) {
  if (!shape_ok(M, N, K)) return false;
  if (epi.ss_in != nullptr) {   // fused RMSNorm consumer: 1/rms from the K / 128 slots of each row
    if (K % 128 != 0 || K > 128 * SS_PARTS || epi.mC > 0 || epi.mode == EPI_RESID || epi.mode == EPI_SPLIT_LERP) return false;
    if ((epi.mode == EPI_STORE || epi.mode == EPI_QKV_ROPE) && N % 128 != 0) return false;
  }
  if (epi.ss_out != nullptr && !rowss_fits(N, epi)) return false;
  if (epi.mC > 0) {   // TokenMerge gather folded into the A loads: 128-wide tiles, plain store epilogue
    int bw, bh;
    if (epi.mode != EPI_STORE || N % 128 != 0 || epi.mC % 64 != 0 || K != 4 * epi.mC || M % epi.mwc != 0 || !quad_box(epi.mwc, &bw, &bh)) return false;
  }
  switch (epi.mode) {
    case EPI_STORE:
    case EPI_RESID:
      return true;
    case EPI_GEGLU:   // 128-wide tiles only
      return N % 128 == 0;
    case EPI_SPLIT_LERP:
      return epi.C % 32 == 0 && N == 4 * epi.C;
    case EPI_QKV_ROPE:
      return N == 3 * epi.C && epi.C % 64 == 0 && epi.nh * 64 == epi.C && epi.rope != nullptr && (epi.rope_r == 32 || epi.rope_r == 64);
    case EPI_PATCH_OUT:   // 48 of 64 columns used; float4 stores of img and loads of x_in
      return N == 64 && epi.W % 4 == 0 && aligned16(epi.img) && (epi.sigma_data <= 0.f || aligned16(epi.x_in));
    default:
      return false;
  }
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

constexpr int PATCH_IN_THREADS = 160;   // warps 0-3: gather + MMA + epilogue, warp 4: weight load
constexpr int PATCH_IN_LD = 132;   // fp32 accumulator row pitch (+4: rows start on different banks)
constexpr size_t PATCH_IN_SMEM = 1024 + 2 * A_STAGE_BYTES + (size_t)BM * PATCH_IN_LD * 4 + 2 * SUB_TILE_BYTES + 64;

__global__ void __launch_bounds__(PATCH_IN_THREADS) patch_in_tc_kernel(const __grid_constant__ CUtensorMap tmw, const __grid_constant__ CUtensorMap tmc,
                                                                   const PatchInParams p) {
  KDB_PDL_TRIGGER();
  constexpr int LD = PATCH_IN_LD;
  uint8_t* sA = tc::smem_1k();              // [128 tokens x 64] bf16, SWIZZLE_128B
  uint8_t* sW = sA + A_STAGE_BYTES;         // [128 outputs x 64]
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
  tc::mbar_wait_nocall(w_full, 0);
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

// KDB200_DISABLE_TC steers the engine's routes away from the tensor-core kernels; an explicit launch_gemm_tc (kdb_gemm_bf16) still runs
bool tc_gemm_supported(int64_t M, int N, int K, const GemmEpi& epi) { return !g_tc_disabled && gemm_fits(M, N, K, epi); }

// true when the RESID / SPLIT / STORE GEMM of this shape runs on 128-wide tiles, which leave sum(x^2) of every row they write
bool tc_gemm_emits_rowss(int64_t M, int N, int K, const GemmEpi& epi) { return tc_gemm_supported(M, N, K, epi) && rowss_fits(N, epi); }

int launch_gemm_tc(const bf16* A, const bf16* W, bf16* C, int64_t M, int N, int K, const GemmEpi& epi, cudaStream_t st) {
  KDB_REQUIRE(aligned16(A) && aligned16(W) && aligned16(C), KDB_ERR_BAD_ARG, "gemm_tc: operands must be 16-byte aligned");
  KDB_REQUIRE(gemm_fits(M, N, K, epi), KDB_ERR_UNSUPPORTED, "gemm_tc: epilogue %d does not support M=%lld N=%d K=%d with these options", epi.mode,
              (long long)M, N, K);
  GemmArgs p{};
  static_cast<GemmEpi&>(p) = epi;
  p.out = C;
  p.M = M;
  p.N = N;
  p.K = K;
  p.th = epi.H / 4;
  p.tw = epi.W / 4;
  if (epi.mC > 0) {
    quad_box(epi.mwc, &p.box_w, &p.box_h);
    return launch_tc<128, EPI_STORE>(A, W, p, st);
  }
  // the split moves its skip and output tiles by TMA when a 128-row block is one box of the quadrant maps (else box_w stays 0).
  // Each tile reads exactly the skip elements it writes, so `out` may alias `skip`.
  if (epi.mode == EPI_SPLIT_LERP && epi.C % 64 == 0 && epi.wc > 0 && M % epi.wc == 0 && aligned16(epi.resid)) quad_box(epi.wc, &p.box_w, &p.box_h);
  switch (epi.mode) {
    case EPI_STORE:
      return dispatch_bn<EPI_STORE>(A, W, p, st);
    case EPI_RESID:
      return dispatch_bn<EPI_RESID>(A, W, p, st);
    case EPI_GEGLU:
      return launch_tc<128, EPI_GEGLU>(A, W, p, st);
    case EPI_SPLIT_LERP:
      return dispatch_bn<EPI_SPLIT_LERP>(A, W, p, st);
    case EPI_QKV_ROPE:
      return epi.rope_r == 64 ? dispatch_bn<EPI_QKV_ROPE, 64>(A, W, p, st) : dispatch_bn<EPI_QKV_ROPE>(A, W, p, st);
    case EPI_PATCH_OUT:
      return launch_tc<64, EPI_PATCH_OUT>(A, W, p, st);
    default:
      return KDB_ERR_BAD_ARG;   // (not reached: gemm_fits accepts no other mode)
  }
}

bool tc_patch_in_supported(const float* x, int C0, int Wimg) {
  return !g_tc_disabled && C0 % 128 == 0 && C0 <= 128 * SS_PARTS && Wimg % 4 == 0 && aligned16(x);
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
  KDB_REQUIRE(tc_patch_in_supported(x, C0, Wimg), KDB_ERR_UNSUPPORTED,
              "patch_in_tc: needs C0 %% 128 == 0, C0 <= %d, W %% 4 == 0 and a 16-byte aligned input (got C0=%d W=%d)", 128 * SS_PARTS, C0, Wimg);
  CUtensorMap tw, tcm;
  int rc;
  if ((rc = tmap_2d(&tw, W_perm, 64, (uint64_t)C0, 64, 128))) return rc;
  if ((rc = tmap_2d(&tcm, out, (uint64_t)C0, (uint64_t)p.M, 64, BM))) return rc;
  static bool opened = false;
  if ((rc = set_smem_once(patch_in_tc_kernel, opened, (int)PATCH_IN_SMEM))) return rc;
  patch_in_tc_kernel<<<dim3((unsigned)ceil_div(p.M, BM), (unsigned)(C0 / 128)), PATCH_IN_THREADS, PATCH_IN_SMEM, st>>>(tw, tcm, p);
  KDB_LAUNCH_CHECK(F_PATCH_IN, st);
  return 0;
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

bool tc_attn_block_supported(int h, int w, int C, int nh, int e, int attn_type, int attn_param, int shift) {
  return !g_tc_disabled && attn_block_supported(h, w, C, nh, e, attn_type, attn_param, shift);
}

int launch_attn_block(bf16* x, const bf16* w_qkv, const bf16* w_out, const float2* rope, const float* qk_scale, int B, int h, int w, int shift,
                      const float* ss_in, float* ss_out, cudaStream_t st) {
  KDB_REQUIRE(B > 0 && attn_block_supported(h, w, AB_C, 2, 64, KDB_ATTN_SHIFTED_WINDOW, 8, shift), KDB_ERR_BAD_SHAPE,
              "attn_block: unsupported shape (needs C = 128, two heads of 64, window 8, shift 0 or 4, h %% 8 == 0, w %% 8 == 0; got B=%d h=%d w=%d shift=%d)",
              B, h, w, shift);
  return launch_attn_block_impl(x, w_qkv, w_out, rope, qk_scale, B, h, w, shift, ss_in, ss_out, st);
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
  GemmEpi e;
  e.mode = EPI_GEGLU;
  e.ss_in = ss_in;
  KDB_REQUIRE(tc_gemm_supported(M, N2, K, e), KDB_ERR_UNSUPPORTED,
              "gemm_bf16_geglu: needs N2 %% 128 == 0 and K %% 64 == 0 (K %% 128 == 0, K <= 1024 with ss_in); got M=%d N2=%d K=%d", M, N2, K);
  return launch_gemm_tc(static_cast<const bf16*>(a), static_cast<const bf16*>(w_il), static_cast<bf16*>(c), M, N2, K, e, (cudaStream_t)stream);
}

extern "C" int kdb_ffn_fused_bf16(void* x, const void* w_up_il, const void* w_down, int M, int d_ff, const float* ss_in, float* ss_out, void* stream) {
  using namespace kdb;
  KDB_REQUIRE(x && w_up_il && w_down && ss_in, KDB_ERR_BAD_ARG, "ffn_fused_bf16: NULL operand");
  return launch_ffn_fused(static_cast<bf16*>(x), static_cast<const bf16*>(w_up_il), static_cast<const bf16*>(w_down), M, 128, d_ff, ss_in, ss_out,
                          (cudaStream_t)stream);
}

extern "C" int kdb_attn_block_bf16(void* x, const void* w_qkv, const void* w_out, const float* rope, const float* qk_scale, int batch, int h, int w,
                                   int shift, const float* ss_in, float* ss_out, void* stream) {
  using namespace kdb;
  KDB_REQUIRE(x && w_qkv && w_out && rope && qk_scale && ss_in && ss_out, KDB_ERR_BAD_ARG, "attn_block_bf16: NULL operand");
  return launch_attn_block(static_cast<bf16*>(x), static_cast<const bf16*>(w_qkv), static_cast<const bf16*>(w_out), reinterpret_cast<const float2*>(rope),
                           qk_scale, batch, h, w, shift, ss_in, ss_out, (cudaStream_t)stream);
}
