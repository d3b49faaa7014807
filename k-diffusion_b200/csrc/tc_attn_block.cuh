// tc_attn_block.cuh -- the whole shifted-window attention block of a 128-wide level in ONE kernel (included inside tc_kernels.cu's
// anonymous namespace).
//
//   x <- x + out_proj( window_attn( rope(cos_sim(q)), rope(cos_sim(k)), v ) ),   [q k v] = AdaRMSNorm(x) . Wqkv^T
//                                                        (reference image_transformer_v2.py:253-337, :106-114, :187-199, :245-248, :396)
//
// Unfused this is three launches (qkv projection, attention, out_proj + residual), each a full HBM round trip of the token stream
// (x -> qkv -> attention output -> x: ~11 bytes moved per byte of x).  Here every 8x8 window is read once and written once; q, k, v and
// the attention output never leave the SM.  Per window (64 tokens) and head h (d_head 64, two heads), all m64 wgmma:
//
//   V, K, Q   = X . Wqkv_h^T          64 x 64 accumulators, A = the X window in shared memory; issued together, the
//                                    v and k epilogues overlap the K and Q MMAs
//   v         : x 1/rms (the row statistics the producer of x left); bf16 -> shared memory (B operand of P V)
//   k, q      : cosine-normalised in registers (a row's 64 columns sit in the 4 threads of a quad: two shfl_xor), x sqrt(scale_h),
//               RoPE from the per-layer table (columns 2i, 2i+1 pair with 16+2i, 17+2i: same thread); k -> shared memory, q stays in
//               registers as the A fragment of S = Q K^T (the accumulator fragment of two 8-column blocks is the A fragment of one k16 step)
//   S = Q K^T : softmax in registers (row max and sum by quad shuffles), seam mask by quadrant as attn_ws_kernel; P is the A operand of
//   O = P V   : O / l -> bf16 A fragment, kept in registers
//
// and after both heads acc = sum_h O_h . Wout[:, 64h:64h+64]^T (wgmma, A from registers), the residual is added from the X tile still in shared memory, sum(x_new^2) is left for the fused RMSNorm of the
// feed-forward block, and the window leaves by TMA from the X buffer itself.  AdaRMSNorm is fused as in the stand-alone GEMMs: Wqkv
// carries the channel scale for this evaluation (fold kernel); q and k are scale invariant, so only v needs 1/rms.
//
// Gather / scatter: a window is four 4x4-token quadrant boxes of a 4-D tensor map over x (C, w, h, B), one box per 64 channels.  The
// roll of the shifted layers (:274) is the quadrants' coordinates; shift 0 uses the same row order.  Rows of a window: quadrant-major,
// then (row, column) inside the quadrant -- the seam-mask regions (:300-315) are whole quadrants.
//
// Roles (384 threads, one CTA per SM, tiles of two windows blockIdx.x, + gridDim.x, ...):
//   warpgroups 0, 1   window 2 tile + wg; the second warpgroup of the last tile idles when the number of windows is odd.  The V, K
//                     and Q accumulators of a head are live together, and the RoPE table entries load under the MMAs
//   warpgroup 2       producer: one elected lane of warp 8 loads by TMA the weights once per CTA, then the X tiles (2 buffers)
// Shared memory: X 2 x 32 KiB, Wqkv 96 KiB, Wout 32 KiB, K and V per warpgroup 4 x 8 KiB = 224 KiB.
#pragma once

constexpr int AB_C = 128;                          // level width this kernel is built for: two heads of 64
constexpr int AB_XBUF = 2;
constexpr int AB_X_BYTES = 2 * A_STAGE_BYTES;      // two windows x 128 channels = two SW128 k-block tiles [128 x 64]
constexpr int AB_WQKV_KB = 3 * AB_C * 128;         // one k-block of Wqkv: [384 rows x 64] bf16 = 48 KiB
constexpr int AB_WO_BYTES = 2 * A_STAGE_BYTES;     // Wout [128 x 128]: k-block h = the input channels of head h
constexpr int AB_KV_BYTES = 64 * 128;              // one [64 tokens x 64] bf16 SW128 tile
constexpr int AB_THREADS = 256 + 128;

struct AttnBlockBars {
  uint64_t w_full;
  tc::TmaRing<AB_XBUF> x;
};
constexpr size_t AB_SMEM = (size_t)AB_XBUF * AB_X_BYTES + 2 * AB_WQKV_KB + AB_WO_BYTES + 4 * AB_KV_BYTES + sizeof(AttnBlockBars) + 1024;

struct AttnBlockParams {
  const float* ss_in;      // [M, SS_PARTS] sum(x^2) of the input rows (slot 0 = the 128 channels)
  float* ss_out;           // same for the output rows
  const float4* rope;      // [2][8][h * w] (cos t_2i, cos t_2i+1, sin t_2i, sin t_2i+1), see rope_table_kernel
  const float* qk_scale;   // [2] cosine-similarity scale per head
  int h, w, shift, nwin;   // nwin = B (h / 8) (w / 8)
};

__global__ void __launch_bounds__(AB_THREADS, 1) gemm_wg_attn_block_kernel(const __grid_constant__ CUtensorMap tmx,
                                                                          const __grid_constant__ CUtensorMap tmwq,
                                                                          const __grid_constant__ CUtensorMap tmwo, const AttnBlockParams p) {
  uint8_t* sX = tc::smem_1k();
  uint8_t* sWQ = sX + AB_XBUF * AB_X_BYTES;
  uint8_t* sWO = sWQ + 2 * AB_WQKV_KB;
  uint8_t* sKV = sWO + AB_WO_BYTES;
  AttnBlockBars* bars = reinterpret_cast<AttnBlockBars*>(sKV + 4 * AB_KV_BYTES);
  const int pwarp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_local = tc::tiles_owned((p.nwin + 1) >> 1);

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmx);
    tc::tma_prefetch_desc(&tmwq);
    tc::tma_prefetch_desc(&tmwo);
    tc::mbar_init(&bars->w_full, 1);
    bars->x.init(tc::REL_THREAD_2WG);          // once its store has read the window
    tc::fence_barrier_init();
  }
  __syncthreads();
  // x and its row statistics come from the kernel before us; the folded Wqkv is rewritten by the fold kernel at the start of every
  // evaluation, so the weights are loaded after the wait as well
  tc::pdl_wait();
  KDB_PDL_TRIGGER();

  if (pwarp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    tc::setmaxnreg_dec<tc::PRODUCER_REGS>();
    if (pwarp == 8 && tc::elect_one()) {
      tc::mbar_arrive_expect_tx(&bars->w_full, 2 * AB_WQKV_KB + AB_WO_BYTES);
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        tc::tma_load_2d(sWQ + kb * AB_WQKV_KB, &tmwq, &bars->w_full, kb * BK, 0);
        tc::tma_load_2d(sWQ + kb * AB_WQKV_KB + 192 * 128, &tmwq, &bars->w_full, kb * BK, 192);
        tc::tma_load_2d(sWO + kb * A_STAGE_BYTES, &tmwo, &bars->w_full, kb * BK, 0);
      }
      PipeState<AB_XBUF> xs{};
      for (int i = 0; i < n_local; ++i, xs.advance()) {
        const int win0 = 2 * ((int)blockIdx.x + i * (int)gridDim.x);
        const int nw = p.nwin - win0 < 2 ? 1 : 2;
        uint64_t* bar = bars->x.acquire(xs, (uint32_t)nw * 2u * AB_KV_BYTES);
        for (int s = 0; s < nw; ++s) {
          int b, wi, wj;
          tc::window_coords(win0 + s, p.h, p.w, b, wi, wj);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            int r, c;
            tc::quad_origin(wi, wj, q, p.h, p.w, p.shift, r, c);
#pragma unroll
            for (int kb = 0; kb < 2; ++kb)
              tc::tma_load_4d(sX + (size_t)xs.slot * AB_X_BYTES + kb * A_STAGE_BYTES + s * AB_KV_BYTES + q * 2048, &tmx, bar, kb * BK, c, r, b);
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ warpgroups: one window each
  tc::setmaxnreg_inc<tc::MMA_REGS>();
  const int wg = pwarp >> 2, t = threadIdx.x & 127;
  const int rw = 16 * (t >> 5) + (lane >> 2);                // this thread's two window rows: rw and rw + 8 (same quadrant)
  const int r0 = 64 * wg + rw;                               // ... as rows of the X tile
  const int cq = 2 * (lane & 3);                             // and its column pair inside every 8-column block
  const int quad = rw >> 4, lr = (rw & 15) >> 2, lc = rw & 3;
  uint8_t* sK = sKV + wg * 2 * AB_KV_BYTES;
  uint8_t* sV = sK + AB_KV_BYTES;
  const uint32_t wq_base = tc::smem_u32(sWQ), wo_base = tc::smem_u32(sWO);
  const uint64_t kdesc = tc::smem_desc_k_sw128(tc::smem_u32(sK));
  const uint64_t vdesc = tc::smem_desc_mn_sw128(tc::smem_u32(sV), 1024, 1024);
  const float sqs[2] = {sqrtf(__ldg(p.qk_scale)), sqrtf(__ldg(p.qk_scale + 1))};
  const int T = p.h * p.w;

  // [64 x 64] accumulator -> bf16 SW128 tile, rows = tokens (K-major B operand of S = Q K^T, MN-major B operand of O = P V)
  auto store_tile = [&](uint8_t* dst, const float (&a)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + tc::sw128_offset(rw, j) + cq * 2) = tc::pack_bf16x2(a[4 * j], a[4 * j + 1]);
      *reinterpret_cast<uint32_t*>(dst + tc::sw128_offset(rw + 8, j) + cq * 2) = tc::pack_bf16x2(a[4 * j + 2], a[4 * j + 3]);
    }
  };
  // q, k: cosine-sim scale (:106-114) + axial RoPE (:187-199) of head hd, rows = image tokens tok0, tok1.  cs[rr][jj] = the RoPE table
  // entry of column pair 8 jj + cq of row rw + 8 rr, the same for q and k (window attention's keys are its queries): loaded once per
  // head, while the projections run.
  auto qk_norm_rope = [&](float (&a)[32], int hd, const float4 (&cs)[2][2]) {
    const float sq = sqs[hd];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s0 = fmaf(a[4 * j], a[4 * j], fmaf(a[4 * j + 1], a[4 * j + 1], s0));
      s1 = fmaf(a[4 * j + 2], a[4 * j + 2], fmaf(a[4 * j + 3], a[4 * j + 3], s1));
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float sc[2] = {sq * rsqrtf(s0 + 1e-6f), sq * rsqrtf(s1 + 1e-6f)};
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int i1 = 4 * jj + 2 * rr, i2 = 4 * (jj + 2) + 2 * rr;     // columns 8 jj + cq (+1) and 16 + 8 jj + cq (+1)
        const float4 c = cs[rr][jj];
        const float x1a = a[i1], x1b = a[i1 + 1], x2a = a[i2], x2b = a[i2 + 1];
        a[i1] = fmaf(x2a, -c.z, x1a * c.x) * sc[rr];
        a[i1 + 1] = fmaf(x2b, -c.w, x1b * c.y) * sc[rr];
        a[i2] = fmaf(x1a, c.z, x2a * c.x) * sc[rr];
        a[i2 + 1] = fmaf(x1b, c.w, x2b * c.y) * sc[rr];
      }
#pragma unroll
    for (int j = 4; j < 8; ++j) {
      a[4 * j] *= sc[0];
      a[4 * j + 1] *= sc[0];
      a[4 * j + 2] *= sc[1];
      a[4 * j + 3] *= sc[1];
    }
  };
  // accumulator fragment [64 x 64] -> bf16 A fragments of its four k16 steps
  auto to_afrag = [](const float (&a)[32], uint32_t (&f)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) f[i] = tc::pack_bf16x2(a[2 * i], a[2 * i + 1]);
  };

  tc::mbar_wait_nocall(&bars->w_full, 0);
  PipeState<AB_XBUF> xs{};
  for (int i = 0; i < n_local; ++i, xs.advance()) {
    const int win = 2 * ((int)blockIdx.x + i * (int)gridDim.x) + wg;
    if (win >= p.nwin) continue;
    int b, wi, wj, qr, qc;
    tc::window_coords(win, p.h, p.w, b, wi, wj);
    tc::quad_origin(wi, wj, quad, p.h, p.w, p.shift, qr, qc);
    const int tok0 = (qr + lr) * p.w + qc + lc, tok1 = tok0 + 2 * p.w;
    const int64_t m0 = (int64_t)b * T + tok0, m1 = (int64_t)b * T + tok1;
    const float rstd0 = rsqrtf(__ldg(p.ss_in + m0 * SS_PARTS) / (float)AB_C + 1e-6f);
    const float rstd1 = rsqrtf(__ldg(p.ss_in + m1 * SS_PARTS) / (float)AB_C + 1e-6f);
    const bool seam_r = p.shift > 0 && wi == 0, seam_c = p.shift > 0 && wj == 0;
    bars->x.wait(xs);
    const uint32_t xa = tc::smem_u32(sX + (size_t)xs.slot * AB_X_BYTES) + (uint32_t)wg * AB_KV_BYTES;   // this window's rows of both k-blocks
    uint32_t of[2][16];                        // O_h / l of both heads: bf16 A fragments of the out projection
#pragma unroll 1
    for (int hd = 0; hd < 2; ++hd) {
      // ---- V, K, Q = X . Wqkv_h^T, three commit groups issued together
      float va[32], ka[32], qa[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) va[j] = ka[j] = qa[j] = 0.f;
      tc::wg_fence_acc(va);
      tc::wg_fence_acc(ka);
      tc::wg_fence_acc(qa);
      tc::wg_fence();
      auto project = [&](float (&d)[32], int third) {      // third: 0 = q, 1 = k, 2 = v (feature order (t nh e))
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint64_t ad = tc::smem_desc_k_sw128(xa + (uint32_t)(kb * A_STAGE_BYTES));
          const uint64_t bd = tc::smem_desc_k_sw128(wq_base + (uint32_t)(kb * AB_WQKV_KB + (third * AB_C + 64 * hd) * 128));
#pragma unroll
          for (int k = 0; k < 4; ++k) tc::wgmma_64<0>(d, ad + 2ull * k, bd + 2ull * k, 1u);
        }
        tc::wg_commit();
      };
      project(va, 2);
      project(ka, 1);
      project(qa, 0);
      float4 cs[2][2];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const float4* tb = p.rope + (int64_t)(hd * 8 + 4 * jj + (lane & 3)) * T;
        cs[0][jj] = __ldg(tb + tok0);
        cs[1][jj] = __ldg(tb + tok1);
      }
      if (hd == 1) tc::named_barrier_sync(tc::BAR_WG + wg, 128);     // head 0's S and P V MMAs (all four warps) are done with K and V
      tc::wg_wait<2>();
      tc::wg_fence_acc(va);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        va[4 * j] *= rstd0;
        va[4 * j + 1] *= rstd0;
        va[4 * j + 2] *= rstd1;
        va[4 * j + 3] *= rstd1;
      }
      store_tile(sV, va);
      tc::wg_wait<1>();
      tc::wg_fence_acc(ka);
      qk_norm_rope(ka, hd, cs);
      store_tile(sK, ka);
      tc::wg_wait<0>();
      tc::wg_fence_acc(qa);
      qk_norm_rope(qa, hd, cs);
      uint32_t qf[16];
      to_afrag(qa, qf);
      tc::fence_proxy_async();                 // K, V (generic-proxy writes) -> visible to the tensor core
      tc::named_barrier_sync(tc::BAR_WG + wg, 128);
      // ---- S = Q K^T
      float s[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) s[j] = 0.f;
      tc::wg_fence_acc(s);
      tc::wg_fence_acc(qf);
      tc::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {qf[4 * kk], qf[4 * kk + 1], qf[4 * kk + 2], qf[4 * kk + 3]};
        tc::wgmma_64_rs<0>(s, a, kdesc + 2ull * kk, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(s);
      // ---- softmax in registers (one key block, unbounded) and O = P V.  Key column block j lies in quadrant j / 2.
      float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;
      float o[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = 0.f;
      auto key_ok = [&](int j) { return tc::seam_ok(quad, j >> 1, seam_r, seam_c); };
      tc::softmax_pv<64, false>(s, key_ok, false, mx0, mx1, l0, l1, o, vdesc);
      tc::softmax_normalize(o, l0, l1);
      uint32_t oh[16];
      to_afrag(o, oh);
#pragma unroll
      for (int j = 0; j < 16; ++j) {          // (register moves under a predicate: of stays out of local memory)
        of[0][j] = hd == 0 ? oh[j] : of[0][j];
        of[1][j] = hd == 0 ? of[1][j] : oh[j];
      }
    }
    // ---- acc = sum_h O_h . Wout[:, 64 h : 64 h + 64]^T, once both heads are done: the 64-register accumulator is not live next to
    // the per-head ones
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    tc::wg_fence_acc(acc);
    tc::wg_fence_acc(of[0]);
    tc::wg_fence_acc(of[1]);
    tc::wg_fence();
#pragma unroll
    for (int hd = 0; hd < 2; ++hd) {
      const uint64_t od = tc::smem_desc_k_sw128(wo_base + (uint32_t)(hd * A_STAGE_BYTES));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {of[hd][4 * kk], of[hd][4 * kk + 1], of[hd][4 * kk + 2], of[hd][4 * kk + 3]};
        tc::wgmma_128_rs(acc, a, od + 2ull * kk, 1u);
      }
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc);
    // ---- epilogue: x_new = acc + x (residual from the X tile in shared memory), in place, then TMA store of this window
    uint8_t* xt = sX + (size_t)xs.slot * AB_X_BYTES;
    const float2 ss = tc::residual_add(xt, r0, cq, acc);
    if ((lane & 3) == 0) {
      p.ss_out[m0 * SS_PARTS] = ss.x;
      p.ss_out[m1 * SS_PARTS] = ss.y;
    }
    tc::fence_proxy_async();
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
    if (t == 0) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int r, c;
        tc::quad_origin(wi, wj, q, p.h, p.w, p.shift, r, c);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) tc::tma_store_4d(&tmx, xt + kb * A_STAGE_BYTES + wg * AB_KV_BYTES + q * 2048, kb * BK, c, r, b);
      }
      tc::tma_store_commit();
      tc::tma_store_wait_read();         // the X buffer may be refilled (tile i + 2)
      bars->x.release(xs);
    }
  }
}

inline bool attn_block_supported(int h, int w, int C, int nh, int e, int attn_type, int attn_param, int shift) {
  return C == AB_C && nh == 2 && e == 64 && attn_type == KDB_ATTN_SHIFTED_WINDOW && attn_param == 8 && (shift == 0 || shift == 4) && h > 0 &&
         w > 0 && h % 8 == 0 && w % 8 == 0;
}

// x [B, h, w, 128] bf16 (raw residual stream, updated IN PLACE), w_qkv [384, 128] (AdaRMSNorm scale folded in), w_out [128, 128],
// rope / qk_scale as AttnBlockParams, ss_in / ss_out [B h w, SS_PARTS] row statistics (may alias)
int launch_attn_block_impl(bf16* x, const bf16* w_qkv, const bf16* w_out, const float2* rope, const float* qk_scale, int B, int h, int w,
                           int shift, const float* ss_in, float* ss_out, cudaStream_t st) {
  CUtensorMap tx, twq, two;
  int rc;
  if ((rc = make_tmap_tokens(&tx, x, AB_C, B, h, w, BK, 4, 4))) return rc;
  if ((rc = tmap_2d(&twq, w_qkv, AB_C, 3 * AB_C, BK, 192))) return rc;
  if ((rc = tmap_2d(&two, w_out, AB_C, AB_C, BK, AB_C))) return rc;
  static bool opened = false;
  if ((rc = set_smem_once(gemm_wg_attn_block_kernel, opened, (int)AB_SMEM))) return rc;
  AttnBlockParams p{ss_in, ss_out, reinterpret_cast<const float4*>(rope), qk_scale, h, w, shift, B * (h / 8) * (w / 8)};
  KDB_CUDA(launch_pdl(gemm_wg_attn_block_kernel, persistent_grid((p.nwin + 1) / 2), dim3(AB_THREADS), AB_SMEM, st, tx, twq, two, p));
  KDB_LAUNCH_CHECK(F_GEMM_TC, st);
  return 0;
}
