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
// Roles (288 threads, one CTA per SM, tiles blockIdx.x, + gridDim.x, ...):
//   warpgroups 0, 1   rows [0, 64) / [64, 128) of every tile: M1, GEGLU, M2, final epilogue; both read the same weight chunks
//   warp 8            TMA producer: X tiles (2 buffers), Wup chunks (3 x 32 KiB ring), Wdown chunks (3 x 16 KiB ring) -- the weights
//                     stream from L2 once per tile (all CTAs walk the same chunks at about the same time)
// Shared memory: X 2 x 32 KiB, Wup 3 x 32 KiB, Wdown 3 x 16 KiB = 208 KiB.
#pragma once

constexpr int FF_C = 128;                  // level width this kernel is built for
constexpr int FF_CH = 64;                  // hidden features per chunk
constexpr int FF_XBUF = 2, FF_WU = 3, FF_WD = 3;
constexpr int FF_X_BYTES = 2 * A_STAGE_BYTES;       // [128 x 128] bf16 = two SW128 k-block tiles
constexpr int FF_WU_BYTES = 2 * A_STAGE_BYTES;      // [128 rows x 128 K]
constexpr int FF_WD_BYTES = A_STAGE_BYTES;          // [128 rows x 64 K]
constexpr int FF_THREADS = 256 + 32;

struct FfnBars {
  uint64_t x_full[FF_XBUF], x_empty[FF_XBUF];
  uint64_t wu_full[FF_WU], wu_empty[FF_WU];
  uint64_t wd_full[FF_WD], wd_empty[FF_WD];
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
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sX = base;
  uint8_t* sWU = sX + FF_XBUF * FF_X_BYTES;
  uint8_t* sWD = sWU + FF_WU * FF_WU_BYTES;
  FfnBars* bars = reinterpret_cast<FfnBars*>(sWD + FF_WD * FF_WD_BYTES);
  const int pwarp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nc = p.nc;
  const int m_tiles = (int)(p.M / BM);
  const int n_local = (int)blockIdx.x < m_tiles ? (m_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmx);
    tc::tma_prefetch_desc(&tmwu);
    tc::tma_prefetch_desc(&tmwd);
    tc::tma_prefetch_desc(&tmo);
    for (int i = 0; i < FF_XBUF; ++i) {
      tc::mbar_init(&bars->x_full[i], 1);
      tc::mbar_init(&bars->x_empty[i], 2);     // one store-drained arrival per warpgroup
    }
    for (int i = 0; i < FF_WU; ++i) {
      tc::mbar_init(&bars->wu_full[i], 1);
      tc::mbar_init(&bars->wu_empty[i], 8);    // lane 0 of each of the eight MMA warps
    }
    for (int i = 0; i < FF_WD; ++i) {
      tc::mbar_init(&bars->wd_full[i], 1);
      tc::mbar_init(&bars->wd_empty[i], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::pdl_wait();                    // x (and its row statistics) come from the kernel before us
  tc::pdl_launch_dependents();

  if (pwarp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (tc::elect_one()) {
      uint32_t su = 0, pu = 0, sd = 0, pd = 0;        // ring slot / phase of the next Wup / Wdown chunk
      for (int i = 0; i < n_local; ++i) {
        const int buf = i & 1;
        tc::mbar_wait(&bars->x_empty[buf], (uint32_t)(((i >> 1) & 1) ^ 1));
        tc::mbar_arrive_expect_tx(&bars->x_full[buf], FF_X_BYTES);
        const int m0 = ((int)blockIdx.x + i * (int)gridDim.x) * BM;
        tc::tma_load_2d(sX + (size_t)buf * FF_X_BYTES, &tmx, &bars->x_full[buf], 0, m0);
        tc::tma_load_2d(sX + (size_t)buf * FF_X_BYTES + A_STAGE_BYTES, &tmx, &bars->x_full[buf], BK, m0);
        for (int c = 0; c < nc; ++c) {
          tc::mbar_wait(&bars->wu_empty[su], pu ^ 1u);
          tc::mbar_arrive_expect_tx(&bars->wu_full[su], FF_WU_BYTES);
          tc::tma_load_2d(sWU + (size_t)su * FF_WU_BYTES, &tmwu, &bars->wu_full[su], 0, c * 128);
          tc::tma_load_2d(sWU + (size_t)su * FF_WU_BYTES + A_STAGE_BYTES, &tmwu, &bars->wu_full[su], BK, c * 128);
          if (++su == FF_WU) {
            su = 0;
            pu ^= 1u;
          }
          tc::mbar_wait(&bars->wd_empty[sd], pd ^ 1u);
          tc::mbar_arrive_expect_tx(&bars->wd_full[sd], FF_WD_BYTES);
          tc::tma_load_2d(sWD + (size_t)sd * FF_WD_BYTES, &tmwd, &bars->wd_full[sd], c * FF_CH, 0);
          if (++sd == FF_WD) {
            sd = 0;
            pd ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ warpgroups: rows [64 wg, 64 wg + 64) of every tile
  const int wg = pwarp >> 2, t = threadIdx.x & 127;
  const int r0 = 64 * wg + 16 * (t >> 5) + (lane >> 2);      // this thread's two accumulator rows: r0 and r0 + 8
  const int cq = 2 * (lane & 3);                             // and its column pair inside every 8-column block
  const uint32_t wu_base = tc::smem_u32(sWU), wd_base = tc::smem_u32(sWD);
  uint32_t su = 0, pu = 0, sd = 0, pd = 0;
  for (int i = 0; i < n_local; ++i) {
    const int buf = i & 1;
    const int64_t m0 = ((int64_t)blockIdx.x + (int64_t)i * gridDim.x) * BM;
    const float rstd0 = rsqrtf(__ldg(p.ss_in + (m0 + r0) * SS_PARTS) / (float)FF_C + 1e-6f);
    const float rstd1 = rsqrtf(__ldg(p.ss_in + (m0 + r0 + 8) * SS_PARTS) / (float)FF_C + 1e-6f);
    // the GELU's 0.5 rides on the value's row scale
    const tc::f32x2 g0 = tc::pk2(rstd0, rstd0), g1 = tc::pk2(rstd1, rstd1), h0 = tc::pk2(0.5f * rstd0, 0.5f * rstd0), h1 = tc::pk2(0.5f * rstd1, 0.5f * rstd1);
    tc::mbar_wait(&bars->x_full[buf], (uint32_t)((i >> 1) & 1));
    const uint32_t xa = tc::smem_u32(sX + (size_t)buf * FF_X_BYTES) + (uint32_t)wg * 8192u;   // rows 64 wg.. of both k-block tiles
    float acc2[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc2[j] = 0.f;
    for (int c = 0; c < nc; ++c) {
      // ---- M1: acc1 = X . Wup_c^T
      float acc1[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc1[j] = 0.f;
      tc::mbar_wait(&bars->wu_full[su], pu);
      const uint32_t wa = wu_base + su * (uint32_t)FF_WU_BYTES;
      tc::wg_fence_acc(acc1);
      tc::wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const uint64_t ad = tc::smem_desc_k_sw128(xa + (uint32_t)(kb * A_STAGE_BYTES)), bd = tc::smem_desc_k_sw128(wa + (uint32_t)(kb * A_STAGE_BYTES));
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_128(acc1, ad + 2ull * k, bd + 2ull * k, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(acc1);
      if (lane == 0) tc::mbar_arrive(&bars->wu_empty[su]);
      if (++su == FF_WU) {
        su = 0;
        pu ^= 1u;
      }
      // ---- GEGLU: 8-column block 2q = 8 value features, block 2q + 1 = their gates -> hidden block q (rows r0, r0 + 8)
      uint32_t hreg[16];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const tc::f32x2 v0 = tc::mul2(tc::pk2(acc1[8 * q], acc1[8 * q + 1]), h0), v1 = tc::mul2(tc::pk2(acc1[8 * q + 2], acc1[8 * q + 3]), h1);
        const tc::f32x2 q0 = tc::mul2(tc::pk2(acc1[8 * q + 4], acc1[8 * q + 5]), g0), q1 = tc::mul2(tc::pk2(acc1[8 * q + 6], acc1[8 * q + 7]), g1);
        float o0, o1, o2, o3;
        tc::upk2(tc::geglu2(v0, q0), o0, o1);
        tc::upk2(tc::geglu2(v1, q1), o2, o3);
        // A fragment of k16 step q / 2: {block 2kk row r0, block 2kk row r0 + 8, block 2kk + 1 row r0, block 2kk + 1 row r0 + 8}
        hreg[(q >> 1) * 4 + (q & 1) * 2 + 0] = tc::pack_bf16x2(o0, o1);
        hreg[(q >> 1) * 4 + (q & 1) * 2 + 1] = tc::pack_bf16x2(o2, o3);
      }
      // ---- M2: acc2 += H_c . Wdown_c^T
      tc::mbar_wait(&bars->wd_full[sd], pd);
      const uint64_t bd = tc::smem_desc_k_sw128(wd_base + sd * (uint32_t)FF_WD_BYTES);
      tc::wg_fence_acc(acc2);
      tc::wg_fence_acc(hreg);
      tc::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {hreg[4 * kk], hreg[4 * kk + 1], hreg[4 * kk + 2], hreg[4 * kk + 3]};
        tc::wgmma_128_rs(acc2, a, bd + 2ull * kk, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(acc2);
      if (lane == 0) tc::mbar_arrive(&bars->wd_empty[sd]);
      if (++sd == FF_WD) {
        sd = 0;
        pd ^= 1u;
      }
    }
    // ---- final epilogue: out = acc2 + x (residual from the X tile in shared memory), in place, then TMA store of this half
    uint8_t* xt = sX + (size_t)buf * FF_X_BYTES;
    float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      uint8_t* sub = xt + (j >> 3) * SUB_TILE_BYTES;
      const uint32_t in16 = (uint32_t)(cq * 2);              // byte offset of the column pair inside its 16-byte chunk
      uint32_t* p0 = reinterpret_cast<uint32_t*>(sub + tc::sw128_offset(r0, j & 7) + in16);
      uint32_t* p1 = reinterpret_cast<uint32_t*>(sub + tc::sw128_offset(r0 + 8, j & 7) + in16);
      const uint32_t x0 = *p0, x1 = *p1;
      const float a0 = acc2[4 * j] + __uint_as_float(x0 << 16), a1 = acc2[4 * j + 1] + __uint_as_float(x0 & 0xffff0000u);
      const float b0 = acc2[4 * j + 2] + __uint_as_float(x1 << 16), b1 = acc2[4 * j + 3] + __uint_as_float(x1 & 0xffff0000u);
      ss0 = fmaf(a0, a0, fmaf(a1, a1, ss0));
      ss1 = fmaf(b0, b0, fmaf(b1, b1, ss1));
      *p0 = tc::pack_bf16x2(a0, a1);
      *p1 = tc::pack_bf16x2(b0, b1);
    }
    ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1);
    ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
    ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1);
    ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
    if (p.ss_out != nullptr && (lane & 3) == 0) {
      p.ss_out[(m0 + r0) * SS_PARTS] = ss0;
      p.ss_out[(m0 + r0 + 8) * SS_PARTS] = ss1;
    }
    tc::fence_proxy_async();
    tc::named_barrier_sync(1 + wg, 128);
    if (t == 0) {
      tc::tma_store_2d(&tmo, xt + wg * 8192, 0, (int)m0 + 64 * wg);
      tc::tma_store_2d(&tmo, xt + SUB_TILE_BYTES + wg * 8192, 64, (int)m0 + 64 * wg);
      tc::tma_store_commit();
      tc::tma_store_wait_read();         // the X buffer may be refilled (tile i + 2)
      tc::mbar_arrive(&bars->x_empty[buf]);
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
  static bool attr_set = false;
  if (!attr_set) {
    KDB_CUDA(cudaFuncSetAttribute(ffn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FF_SMEM));
    attr_set = true;
  }
  static const bool no_pdl = [] {
    const char* e = getenv("KDB200_NO_PDL");
    return e != nullptr && e[0] == '1';
  }();
  FfnParams p{ss_in, ss_out, M, dff / FF_CH};
  const int64_t m_tiles = M / BM;
  cudaLaunchConfig_t lc{};
  lc.gridDim = dim3((unsigned)(m_tiles < num_sms() ? m_tiles : num_sms()));
  lc.blockDim = dim3(FF_THREADS);
  lc.dynamicSmemBytes = FF_SMEM;
  lc.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = attr;
  lc.numAttrs = no_pdl ? 0 : 1;
  KDB_CUDA(cudaLaunchKernelEx(&lc, ffn_fused_kernel, tx, twu, twd, to, p));
  KDB_LAUNCH_CHECK(F_GEMM_TC, st);
  return 0;
}
