// tc_ffn_fused.cuh -- the whole feed-forward block of a 128-wide level in ONE kernel (included inside tc_kernels.cu's anonymous namespace).
//
//   x <- x + down_proj( value(x_n) * gelu(gate(x_n)) ),   x_n = AdaRMSNorm(x)            (reference image_transformer_v2.py:479-493, :89-95)
//
// Unfused this is two launches: up_proj + GEGLU writes the [M, d_ff] hidden to HBM and down_proj reads it back.  Here the hidden never
// leaves the registers: per 128-token tile the CTA walks d_ff in chunks of 64 hidden features,
//
//   M1(c):  acc1     = X[64 x C] . Wup_c^T           128 accumulator columns = 8 x (8 value | 8 gate) features, K = C      (wgmma, A and B in smem)
//   G(c):   H_c      = value * gelu(gate) * ...      in registers: a value column and its gate column sit in the same thread
//   M2(c):  acc2    += H_c[64 x 64] . Wdown_c^T      H_c is the A operand straight from registers (the accumulator fragment of
//                                                    two 8-column blocks is the bf16 A fragment of one k16 step), K = 64
//
// and after the last chunk the residual is added (the X tile is still in shared memory), sum(x^2) is left for the next fused RMSNorm,
// and the tile is stored by TMA from the X buffer itself.  AdaRMSNorm is fused as in the stand-alone GEMMs: Wup carries the channel scale
// for this evaluation (fold kernel), 1/rms of the row comes from the statistics its producer left.
//
// Roles (384 threads, one CTA per SM, tiles blockIdx.x, + gridDim.x, ...):
//   warpgroups 0, 1   rows [0, 64) / [64, 128) of every tile: M1, GEGLU, M2, final epilogue; both read the same weight chunks
//   warpgroup 2       producer: one elected lane of warp 8 streams by TMA the X tiles (2 buffers), Wup chunks (3 x 32 KiB ring),
//                     Wdown chunks (3 x 16 KiB ring) -- the weights from L2 once per tile (all CTAs walk the same chunks together)
// Shared memory: X 2 x 32 KiB, Wup 3 x 32 KiB, Wdown 3 x 16 KiB = 208 KiB.
//
// Schedule: a warpgroup issues its MMAs in blocks -- M1(0) of a tile, then after each GEGLU(c) the block M2(c), M1(c + 1) -- and the two
// warpgroups take turns to issue (BAR_TURN), so that one warpgroup's GEGLU and wait latencies run while the tensor cores
// work through the other's block.  Issued together both would finish together, and the tensor cores would idle during every GEGLU.  A
// warpgroup is at most one block ahead of the other, which the 3-deep weight rings cover.  Every accumulator sees the same wgmma
// sequence as in a serial M1 -> GEGLU -> M2 order: the schedule changes no result bit.
#pragma once

constexpr int FF_C = 128;                  // level width this kernel is built for
constexpr int FF_CH = 64;                  // hidden features per chunk
constexpr int FF_XBUF = 2, FF_WU = 3, FF_WD = 3;
constexpr int FF_X_BYTES = 2 * A_STAGE_BYTES;       // [128 x 128] bf16 = two SW128 k-block tiles
constexpr int FF_WU_BYTES = 2 * A_STAGE_BYTES;      // [128 rows x 128 K]
constexpr int FF_WD_BYTES = A_STAGE_BYTES;          // [128 rows x 64 K]
constexpr int FF_THREADS = 256 + 128;

struct FfnBars {
  tc::TmaRing<FF_XBUF> x;
  tc::TmaRing<FF_WU> wu;
  tc::TmaRing<FF_WD> wd;
};
constexpr size_t FF_SMEM = (size_t)FF_XBUF * FF_X_BYTES + (size_t)FF_WU * FF_WU_BYTES + (size_t)FF_WD * FF_WD_BYTES + sizeof(FfnBars) + 1024;

struct FfnParams {
  const float* ss_in;      // [M, SS_PARTS] sum(x^2) of the input rows (slot 0 = the 128 channels)
  float* ss_out;           // same for the output rows, or nullptr
  int64_t M;               // tokens, multiple of 128
  int nc;                  // d_ff / 64 chunks
};

__global__ void __launch_bounds__(FF_THREADS, 1) ffn_fused_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmwu,
                                                                 const __grid_constant__ CUtensorMap tmwd, const __grid_constant__ CUtensorMap tmo,
                                                                 const FfnParams p) {
  uint8_t* sX = tc::smem_1k();
  uint8_t* sWU = sX + FF_XBUF * FF_X_BYTES;
  uint8_t* sWD = sWU + FF_WU * FF_WU_BYTES;
  FfnBars* bars = reinterpret_cast<FfnBars*>(sWD + FF_WD * FF_WD_BYTES);
  const int pwarp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nc = p.nc;
  const int n_local = tc::tiles_owned((int)(p.M / BM));

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmx);
    tc::tma_prefetch_desc(&tmwu);
    tc::tma_prefetch_desc(&tmwd);
    tc::tma_prefetch_desc(&tmo);
    bars->x.init(tc::REL_THREAD_2WG);          // once its store has read the tile
    bars->wu.init(tc::REL_WARPS_2WG);
    bars->wd.init(tc::REL_WARPS_2WG);
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::pdl_wait();                    // x (and its row statistics) come from the kernel before us
  KDB_PDL_TRIGGER();

  if (pwarp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    tc::setmaxnreg_dec<tc::PRODUCER_REGS>();
    if (pwarp == 8 && tc::elect_one()) {
      PipeState<FF_XBUF> xs{};
      PipeState<FF_WU> us{};
      PipeState<FF_WD> ds{};
      for (int i = 0; i < n_local; ++i, xs.advance()) {
        uint64_t* bar = bars->x.acquire(xs, FF_X_BYTES);
        const int m0 = ((int)blockIdx.x + i * (int)gridDim.x) * BM;
        tc::tma_load_2d(sX + (size_t)xs.slot * FF_X_BYTES, &tmx, bar, 0, m0);
        tc::tma_load_2d(sX + (size_t)xs.slot * FF_X_BYTES + A_STAGE_BYTES, &tmx, bar, BK, m0);
        for (int c = 0; c < nc; ++c, us.advance(), ds.advance()) {
          bar = bars->wu.acquire(us, FF_WU_BYTES);
          tc::tma_load_2d(sWU + (size_t)us.slot * FF_WU_BYTES, &tmwu, bar, 0, c * 128);
          tc::tma_load_2d(sWU + (size_t)us.slot * FF_WU_BYTES + A_STAGE_BYTES, &tmwu, bar, BK, c * 128);
          bar = bars->wd.acquire(ds, FF_WD_BYTES);
          tc::tma_load_2d(sWD + (size_t)ds.slot * FF_WD_BYTES, &tmwd, bar, c * FF_CH, 0);
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ warpgroups: rows [64 wg, 64 wg + 64) of every tile
  tc::setmaxnreg_inc<tc::MMA_REGS>();
  const int wg = pwarp >> 2, t = threadIdx.x & 127;
  const int r0 = 64 * wg + 16 * (t >> 5) + (lane >> 2);      // this thread's two accumulator rows: r0 and r0 + 8
  const int cq = 2 * (lane & 3);                             // and its column pair inside every 8-column block
  const uint32_t wu_base = tc::smem_u32(sWU), wd_base = tc::smem_u32(sWD);
  PipeState<FF_XBUF> xs{};
  PipeState<FF_WU> us{};
  PipeState<FF_WD> ds{};
  // Issue turns: warpgroup 0 issues block k after warpgroup 1 has issued block k - 1 (BAR_TURN), warpgroup 1 issues block k after
  // warpgroup 0 has issued block k (BAR_TURN + 1).  Both issue nc + 1 blocks per tile; the arrivals match the syncs one for one.
  bool first_block = true;
  float acc1[64], acc2[64];
  uint32_t hreg[16];
  for (int i = 0; i < n_local; ++i, xs.advance()) {
    const int64_t m0 = ((int64_t)blockIdx.x + (int64_t)i * gridDim.x) * BM;
    const float rstd0 = rsqrtf(__ldg(p.ss_in + (m0 + r0) * SS_PARTS) / (float)FF_C + 1e-6f);
    const float rstd1 = rsqrtf(__ldg(p.ss_in + (m0 + r0 + 8) * SS_PARTS) / (float)FF_C + 1e-6f);
    // the GELU's 0.5 rides on the value's row scale
    const tc::f32x2 g0 = tc::pk2(rstd0, rstd0), g1 = tc::pk2(rstd1, rstd1), h0 = tc::pk2(0.5f * rstd0, 0.5f * rstd0), h1 = tc::pk2(0.5f * rstd1, 0.5f * rstd1);
    bars->x.wait(xs);
    const uint32_t xa = tc::smem_u32(sX + (size_t)xs.slot * FF_X_BYTES) + (uint32_t)wg * 8192u;   // rows 64 wg.. of both k-block tiles
#pragma unroll
    for (int j = 0; j < 64; ++j) acc2[j] = 0.f;
    // block c: M2(c - 1) for c > 0, M1(c) for c < nc.  One program point per wgmma: accumulators carried into the loop from a second
    // issue site would take register moves inside the in-flight stage, and ptxas would serialise the wgmmas.
    for (int c = 0; c <= nc; ++c) {
      if (c > 0) {
        // M1(c - 1) and, from c = 2 on, M2(c - 2) were this warpgroup's last block
        tc::wg_wait<0>();
        tc::wg_fence_acc(acc1);
        tc::wg_fence_acc(acc2);
        tc::wg_fence_acc(hreg);
        if (lane == 0) bars->wu.release(us);
        us.advance();
        if (c > 1) {
          if (lane == 0) bars->wd.release(ds);
          ds.advance();
        }
        // ---- GEGLU(c - 1) -> hidden block q of rows r0, r0 + 8 = the A fragment of M2's k16 steps
        tc::geglu_fragment(acc1, h0, h1, g0, g1, hreg);
      }
#pragma unroll
      for (int j = 0; j < 64; ++j) acc1[j] = 0.f;
      tc::wg_fence_acc(acc1);          // the zeros are written before this turn's first wgmma
      // ---- this warpgroup's turn to issue
      if (wg == 1) tc::named_barrier_sync(tc::BAR_TURN + 1, 256);
      else if (!first_block) tc::named_barrier_sync(tc::BAR_TURN, 256);
      first_block = false;
      if (c > 0) {
        // ---- M2(c - 1): acc2 += H . Wdown^T
        bars->wd.wait(ds);
        const uint64_t bd = tc::smem_desc_k_sw128(wd_base + ds.slot * (uint32_t)FF_WD_BYTES);
        tc::wg_fence_acc(acc2);
        tc::wg_fence_acc(hreg);
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint32_t a[4] = {hreg[4 * kk], hreg[4 * kk + 1], hreg[4 * kk + 2], hreg[4 * kk + 3]};
          tc::wgmma_128_rs(acc2, a, bd + 2ull * kk, 1u);
        }
        tc::wg_commit();
      }
      if (c < nc) {
        // ---- M1(c): acc1 = X . Wup^T
        bars->wu.wait(us);
        const uint32_t wa = wu_base + us.slot * (uint32_t)FF_WU_BYTES;
        tc::wg_fence_acc(acc1);
        tc::wg_fence();
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint64_t ad = tc::smem_desc_k_sw128(xa + (uint32_t)(kb * A_STAGE_BYTES)), bd = tc::smem_desc_k_sw128(wa + (uint32_t)(kb * A_STAGE_BYTES));
#pragma unroll
          for (int k = 0; k < 4; ++k) tc::wgmma_128(acc1, ad + 2ull * k, bd + 2ull * k, 1u);
        }
        tc::wg_commit();
      }
      if (wg == 0) tc::named_barrier_arrive(tc::BAR_TURN + 1, 256);
      else if (c < nc || i + 1 < n_local) tc::named_barrier_arrive(tc::BAR_TURN, 256);
    }
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc2);
    tc::wg_fence_acc(hreg);
    if (lane == 0) bars->wd.release(ds);
    ds.advance();
    // ---- final epilogue: out = acc2 + x (residual from the X tile in shared memory), in place, then TMA store of this half
    uint8_t* xt = sX + (size_t)xs.slot * FF_X_BYTES;
    const float2 ss = tc::residual_add(xt, r0, cq, acc2);
    if (p.ss_out != nullptr && (lane & 3) == 0) {
      p.ss_out[(m0 + r0) * SS_PARTS] = ss.x;
      p.ss_out[(m0 + r0 + 8) * SS_PARTS] = ss.y;
    }
    tc::fence_proxy_async();
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
    if (t == 0) {
      tc::tma_store_2d(&tmo, xt + wg * 8192, 0, (int)m0 + 64 * wg);
      tc::tma_store_2d(&tmo, xt + SUB_TILE_BYTES + wg * 8192, 64, (int)m0 + 64 * wg);
      tc::tma_store_commit();
      tc::tma_store_wait_read();         // the X buffer may be refilled (tile i + 2)
      bars->x.release(xs);
    }
  }
}

// x [M, 128] bf16 (raw residual stream, updated IN PLACE), w_up_il [2 d_ff, 128] (value / gate rows interleaved, AdaRMSNorm scale folded in),
// w_down [128, d_ff], ss_in / ss_out [M, SS_PARTS] row statistics
inline bool ffn_fused_supported(int64_t M, int C, int dff) { return C == FF_C && M > 0 && M % BM == 0 && dff % FF_CH == 0 && dff / FF_CH >= 3; }

int launch_ffn_fused_impl(bf16* x, const bf16* w_up_il, const bf16* w_down, int64_t M, int dff, const float* ss_in, float* ss_out, cudaStream_t st) {
  CUtensorMap tx, twu, twd, to;
  int rc;
  if ((rc = tmap_2d(&tx, x, FF_C, (uint64_t)M, BK, BM))) return rc;
  if ((rc = tmap_2d(&twu, w_up_il, FF_C, (uint64_t)2 * dff, BK, 128))) return rc;
  if ((rc = tmap_2d(&twd, w_down, (uint64_t)dff, FF_C, BK, FF_C))) return rc;
  if ((rc = tmap_2d(&to, x, FF_C, (uint64_t)M, 64, BM / 2))) return rc;     // each warpgroup stores its 64 rows
  static bool opened = false;
  if ((rc = set_smem_once(ffn_fused_kernel, opened, (int)FF_SMEM))) return rc;
  FfnParams p{ss_in, ss_out, M, dff / FF_CH};
  KDB_CUDA(launch_pdl(ffn_fused_kernel, persistent_grid(M / BM), dim3(FF_THREADS), FF_SMEM, st, tx, twu, twd, to, p));
  KDB_LAUNCH_CHECK(F_GEMM_TC, st);
  return 0;
}
