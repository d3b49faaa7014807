// tc_attention.cu -- bf16 attention on the sm_90a tensor core (wgmma) for the attention types of the model configurations:
//   * shifted-window attention, 8x8 windows, d_head 64 (reference image_transformer_v2.py:253-337,446-476)
//   * global attention, sequence a multiple of 128, d_head 64 (:355-396)
//   * 7x7 neighbourhood attention, d_head 64 (:399-443)
// q and k arrive already cosine-normalised and rotated (qknorm_rope kernel); softmax scale is 1.0.
//
// WINDOW and GLOBAL: attn_ws_kernel, persistent and warp-specialized (384 threads, one CTA per SM, tiles blockIdx.x, + gridDim.x, ...).
//   A tile is 128 query rows, 64 per MMA warpgroup, and a sequence of key blocks:
//   WINDOW : the tile is two work items (image, window, head) -- heads 2k and 2k + 1 of one window, one per warpgroup; each warpgroup
//            computes its own 64x64 S with m64n64k16 against its head's 64 keys, one key block.  The roll (:274) is pure index
//            arithmetic: a window is fetched as four 4x4-token TMA boxes (quadrants), which are exactly the seam-mask regions (:300-315);
//            rows of a window are quadrant-major, then (row, column) inside the quadrant.
//   GLOBAL : the tile is 128 queries of one (image, head); keys and values are streamed in blocks of 128 through a ring of stages that
//            both warpgroups read (S = 64 x 128 per warpgroup, m64n128k16).
//   Roles: warpgroup 2 is the producer: one elected lane loads by TMA the Q tile of every tile (WS_QBUF buffers) and its key blocks
//   (WS_KV_STAGES stages of K and V), so the next tile loads while the current one computes.  Warpgroups 0 and 1: S = Q K^T into
//   registers, softmax in registers (a row's columns sit in the 4 threads of a quad: max and sum by two shuffles), P rounded to bf16
//   is the register A operand of O += P V (V an MN-major operand straight from the TMA tile), O stays in registers across the key
//   blocks and is scaled by 1/l once; the bf16 output is staged in shared memory and leaves by TMA (the quadrant boxes for windows).
//   Softmax: with the bound (below) a single pass with the fixed shift exp(s - bound); without it the row maximum: GLOBAL keeps a running
//   maximum and rescales O and l when it grows (exact: the result is that of the final maximum), WINDOW has one key block.
// NA: attn_na_kernel, one CTA = one 128-query block of one head (160 threads).  7x7 neighbourhood (NATTEN definition: window clamped
//   inward at the borders, always 49 keys).  Rows = an 8x16 query block; its keys all lie in the clamped 14x22 halo, streamed as three
//   TMA boxes of 5 halo rows (110 keys per 128-row tile, the tail rows are masked / zero); the per-query 7x7 window is a mask on S.
//   Roles: warp 4 = TMA producer, warps 0-3 = the warpgroup that issues the MMAs and runs the softmax.  Per key block: TMA (SWIZZLE_128B)
//   -> S = Q K^T (wgmma, two M = 64 halves) -> fp32 S tile in shared memory -> softmax (one thread per row) -> P (bf16) written to shared
//   memory in the K-major SW128 layout -> O += P V -> fp32 O tile, 1/l scaling, store.  Without the bound an exact two-pass softmax
//   (pass A: row maxima, pass B: exp / P V).
#include "tc_common.cuh"
#include "tc_kernels.cuh"

namespace kdb {
namespace {

constexpr int ROWS = 128, DH = 64;
constexpr int TILE_BYTES = ROWS * DH * 2;    // 16 KiB: 128 rows x 128 B
constexpr int HALF_BYTES = TILE_BYTES / 2;   // 64 rows: one warpgroup's share, one window of one head
constexpr float LOG2E = 1.4426950408889634f;
constexpr int S_LD = ROWS + 4;               // row pitch (floats) of the fp32 S / O tile

enum { MODE_WINDOW = 0, MODE_GLOBAL = 1 };

constexpr int NA_QH = 8, NA_QW = 16;          // query block of one CTA (128 queries of one head)
constexpr int NA_KH = 14, NA_KW = 22;         // its clamped key halo for a 7x7 neighbourhood
constexpr int NA_BLK_ROWS = 5;                // halo rows per key block: 5 x 22 = 110 keys (of a 128-row tile)
constexpr int NA_BLK_KEYS = NA_BLK_ROWS * NA_KW;

struct AttnParams {
  bf16* out;
  // [nh] or nullptr: upper bound of |q . k| per head.  q and k are cosine-normalised (|q| = |k| = sqrt(scale_h), reference
  // :106-114, RoPE is a rotation), so the layer's scale IS that bound and softmax can use it as a FIXED shift: exp(s - bound)
  // needs no row maximum -> one pass over the key blocks, no maximum scan.
  const float* bound;
  int B, h, w, nh, shift, nblk;
  int n_tiles;                                 // attn_ws_kernel: WINDOW B (h / 8) (w / 8) nh / 2, GLOBAL B nh (h w / 128)
};

// ================================================================ WINDOW, GLOBAL
constexpr int WS_THREADS = 384;
// Loads are the bound (a window tile is ~0.5 us of MMA and softmax against 48 KiB in, 16 KiB out): four tiles in flight per SM keep
// enough bytes outstanding to cover the latency of HBM at its bandwidth share of one SM
constexpr int WS_QBUF = 4, WS_KV_STAGES = 4;

struct WsBars {
  tc::TmaRing<WS_QBUF> q;
  tc::TmaRing<WS_KV_STAGES> kv;
};
// Q buffers, K and V stages, one output staging tile per warpgroup
constexpr size_t WS_SMEM = (size_t)WS_QBUF * TILE_BYTES + (size_t)WS_KV_STAGES * 2 * TILE_BYTES + 2 * HALF_BYTES + sizeof(WsBars) + 1024;

// tile -> image b, window (wi, wj), first head of the pair
__device__ __forceinline__ void ws_window(const AttnParams& p, int tile, int& b, int& wi, int& wj, int& head0) {
  const int hp = p.nh >> 1, win = tile / hp;
  head0 = 2 * (tile - win * hp);
  tc::window_coords(win, p.h, p.w, b, wi, wj);
}
// tile -> image b, head, 128-query tile m (GLOBAL)
__device__ __forceinline__ void ws_global(const AttnParams& p, int tile, int& b, int& head, int& m) {
  b = tile / (p.nh * p.nblk);
  const int rem = tile - b * p.nh * p.nblk;
  head = rem / p.nblk;
  m = rem - head * p.nblk;
}

template <int MODE, bool BOUNDED>
__global__ void __launch_bounds__(WS_THREADS, 1) attn_ws_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_out,
                                                                const AttnParams p) {
  constexpr int NK = MODE == MODE_WINDOW ? 64 : 128;   // keys per block seen by one warpgroup
  uint8_t* sQ = tc::smem_1k();
  uint8_t* sKV = sQ + WS_QBUF * TILE_BYTES;                    // stage s: K at 2 s TILE_BYTES, V after it
  uint8_t* sO = sKV + WS_KV_STAGES * 2 * TILE_BYTES;
  WsBars* bars = reinterpret_cast<WsBars*>(sO + 2 * HALF_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nblk = MODE == MODE_WINDOW ? 1 : p.nblk;
  const int n_local = tc::tiles_owned(p.n_tiles);

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tm_in);
    tc::tma_prefetch_desc(&tm_out);
    bars->q.init(tc::REL_WARPS_2WG);
    bars->kv.init(tc::REL_WARPS_2WG);
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::pdl_wait();                              // programmatic launch: the qkv projection before us must be complete from here on
  KDB_PDL_TRIGGER();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    tc::setmaxnreg_dec<tc::PRODUCER_REGS>();
    if (warp == 8 && tc::elect_one()) {
      // the window of heads head0, head0 + 1, third t of qkv (0 q, 1 k, 2 v): two 64-row halves of four quadrant boxes
      auto load_window = [&](uint8_t* dst, int t, uint64_t* bar, int b, int wi, int wj, int head0) {
#pragma unroll
        for (int hd = 0; hd < 2; ++hd)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            int r, c;
            tc::quad_origin(wi, wj, q, p.h, p.w, p.shift, r, c);
            tc::tma_load_4d(dst + hd * HALF_BYTES + q * 2048, &tm_in, bar, (t * p.nh + head0 + hd) * DH, c, r, b);
          }
      };
      PipeState<WS_QBUF> qs{};
      PipeState<WS_KV_STAGES> ks{};
      for (int i = 0; i < n_local; ++i, qs.advance()) {
        const int tile = (int)blockIdx.x + i * (int)gridDim.x;
        int b, head, wi = 0, wj = 0, m = 0;
        if constexpr (MODE == MODE_WINDOW) ws_window(p, tile, b, wi, wj, head);
        else ws_global(p, tile, b, head, m);
        uint64_t* bar = bars->q.acquire(qs, TILE_BYTES);
        if constexpr (MODE == MODE_WINDOW) load_window(sQ + qs.slot * TILE_BYTES, 0, bar, b, wi, wj, head);
        else tc::tma_load_3d(sQ + qs.slot * TILE_BYTES, &tm_in, bar, head * DH, m * ROWS, b);
        for (int j = 0; j < nblk; ++j, ks.advance()) {     // WINDOW: one key block
          bar = bars->kv.acquire(ks, 2 * TILE_BYTES);
          uint8_t* k_dst = sKV + ks.slot * 2 * TILE_BYTES;
          if constexpr (MODE == MODE_WINDOW) {
            load_window(k_dst, 1, bar, b, wi, wj, head);
            load_window(k_dst + TILE_BYTES, 2, bar, b, wi, wj, head);
          } else {
            tc::tma_load_3d(k_dst, &tm_in, bar, (p.nh + head) * DH, j * ROWS, b);
            tc::tma_load_3d(k_dst + TILE_BYTES, &tm_in, bar, (2 * p.nh + head) * DH, j * ROWS, b);
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ MMA warpgroups: 64 query rows each
  tc::setmaxnreg_inc<tc::MMA_REGS>();
  const int wg = warp >> 2, t = threadIdx.x & 127;
  const int rw = 16 * (t >> 5) + (lane >> 2);                // this thread's two rows of the warpgroup's 64: rw and rw + 8
  const int cq = 2 * (lane & 3);                             // and its column pair inside every 8-column block
  const int quad = rw >> 4;                                  // WINDOW: the quadrant of both rows
  uint8_t* sOw = sO + wg * HALF_BYTES;
  PipeState<WS_QBUF> qs{};
  PipeState<WS_KV_STAGES> ks{};
  for (int i = 0; i < n_local; ++i, qs.advance()) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    int b, head, wi = 0, wj = 0, m = 0;
    if constexpr (MODE == MODE_WINDOW) {
      ws_window(p, tile, b, wi, wj, head);
      head += wg;
    } else {
      ws_global(p, tile, b, head, m);
    }
    const bool seam_r = MODE == MODE_WINDOW && p.shift > 0 && wi == 0;
    const bool seam_c = MODE == MODE_WINDOW && p.shift > 0 && wj == 0;
    float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running row maxima (or the bound) and partial row sums
    if constexpr (BOUNDED) mx0 = mx1 = __ldg(p.bound + head);
    float o[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) o[j] = 0.f;
    const uint64_t qdesc = tc::smem_desc_k_sw128(tc::smem_u32(sQ + qs.slot * TILE_BYTES + wg * HALF_BYTES));
    bars->q.wait(qs);
    for (int j = 0; j < nblk; ++j, ks.advance()) {
      const uint32_t k_addr = tc::smem_u32(sKV + ks.slot * 2 * TILE_BYTES) + (MODE == MODE_WINDOW ? wg * HALF_BYTES : 0);
      const uint32_t v_addr = k_addr + TILE_BYTES;
      bars->kv.wait(ks);
      // ---- S = Q K^T
      float s[NK / 2];
#pragma unroll
      for (int c = 0; c < NK / 2; ++c) s[c] = 0.f;
      tc::wg_fence_acc(s);
      tc::wg_fence();
      const uint64_t kdesc = tc::smem_desc_k_sw128(k_addr);
#pragma unroll
      for (int k = 0; k < DH / 16; ++k) {
        if constexpr (NK == 64)
          tc::wgmma_64<0>(s, qdesc + 2ull * k, kdesc + 2ull * k, 1u);
        else
          tc::wgmma_128(s, qdesc + 2ull * k, kdesc + 2ull * k, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(s);
      if (j == nblk - 1 && lane == 0) bars->q.release(qs);   // every read of this Q tile is done
      // ---- softmax in registers and O += P V.  WINDOW: key column block c lies in quadrant c / 2.
      auto key_ok = [&](int c) { return tc::seam_ok(quad, c >> 1, seam_r, seam_c); };
      tc::softmax_pv<NK, BOUNDED>(s, key_ok, j > 0, mx0, mx1, l0, l1, o, tc::smem_desc_mn_sw128(v_addr, 1024, 1024));
      if (lane == 0) bars->kv.release(ks);
    }
    // ---- O / l -> bf16 staging tile (rows = this warpgroup's 64 queries) -> TMA store
    tc::softmax_normalize(o, l0, l1);
    if (t == 0) tc::tma_store_wait_read();    // the previous tile's store has read the staging tile
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      *reinterpret_cast<uint32_t*>(sOw + tc::sw128_offset(rw, c) + cq * 2) = tc::pack_bf16x2(o[4 * c], o[4 * c + 1]);
      *reinterpret_cast<uint32_t*>(sOw + tc::sw128_offset(rw + 8, c) + cq * 2) = tc::pack_bf16x2(o[4 * c + 2], o[4 * c + 3]);
    }
    tc::fence_proxy_async();                   // staging tile (generic-proxy writes) -> visible to the TMA engine
    tc::named_barrier_sync(tc::BAR_WG + wg, 128);
    if (t == 0) {
      if constexpr (MODE == MODE_WINDOW) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          int r, c;
          tc::quad_origin(wi, wj, q, p.h, p.w, p.shift, r, c);
          tc::tma_store_4d(&tm_out, sOw + q * 2048, head * DH, c, r, b);
        }
      } else {
        tc::tma_store_3d(&tm_out, sOw, head * DH, m * ROWS + wg * 64, b);
      }
      tc::tma_store_commit();
    }
  }
  if (t == 0) tc::tma_store_wait_read();      // shared memory stays alive until the last store has read it
}

// ================================================================ NA
struct Bars {
  uint64_t q;
  tc::TmaRing<1> kv;
};

template <bool BOUNDED>
__global__ void __launch_bounds__(160, 1) attn_na_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_kv,
                                                         const AttnParams p) {
  uint8_t* base = tc::smem_1k();
  uint8_t* sQ = base;
  uint8_t* sK = base + TILE_BYTES;
  uint8_t* sV = base + 2 * TILE_BYTES;
  uint8_t* sP = base + 3 * TILE_BYTES;         // P: two K-blocks of 64 keys, 32 KiB
  float* sS = reinterpret_cast<float*>(base + 5 * TILE_BYTES);   // fp32 S (then O) tile, row pitch S_LD
  Bars* bars = reinterpret_cast<Bars*>(sS + ROWS * S_LD);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nh = p.nh;
  // work decomposition: query block origin and clamped halo origin
  const int b = blockIdx.z, head0 = blockIdx.y;
  const int nbw = p.w / NA_QW;
  const int qi0 = (blockIdx.x / nbw) * NA_QH;
  const int qj0 = (blockIdx.x % nbw) * NA_QW;
  const int r0 = min(max(qi0 - 3, 0), p.h - NA_KH);
  const int c0 = min(max(qj0 - 3, 0), p.w - NA_KW);
  const int nblk = p.nblk;
  constexpr bool bounded = BOUNDED;
  const bool two_pass = nblk > 1 && !bounded;
  const int n_iter = two_pass ? 2 * nblk : nblk;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmap);
    tc::mbar_init(&bars->q, 1);
    bars->kv.init(tc::REL_WARPS);
    tc::fence_barrier_init();
  }
  // rows 110..127 of the V tile are never written by TMA: they must be finite (P there is exactly 0)
  for (int i = threadIdx.x; i < (ROWS - NA_BLK_KEYS) * 8; i += blockDim.x)
    *reinterpret_cast<uint4*>(sV + NA_BLK_KEYS * 128 + i * 16) = make_uint4(0u, 0u, 0u, 0u);
  tc::fence_proxy_async();
  __syncthreads();
  tc::pdl_wait();                              // programmatic launch: the qkv projection before us must be complete from here on
  KDB_PDL_TRIGGER();

  if (warp == 4) {
    if (tc::elect_one()) {
      // ------------------------------------------------ loads of Q and of each key block (K, and V in the P V pass)
      tc::mbar_arrive_expect_tx(&bars->q, TILE_BYTES);
      tc::tma_load_4d(sQ, &tmap, &bars->q, head0 * DH, qj0, qi0, b);
      for (int it = 0; it < n_iter; ++it) {
        const int j = it % nblk;
        const bool with_v = !two_pass || it >= nblk;
        constexpr uint32_t KV_BYTES = NA_BLK_KEYS * 128;
        uint64_t* bar = bars->kv.acquire(PipeState<1>::at(it), with_v ? 2 * KV_BYTES : KV_BYTES);
        tc::tma_load_4d(sK, &tmap_kv, bar, (nh + head0) * DH, c0, r0 + j * NA_BLK_ROWS, b);
        if (with_v) tc::tma_load_4d(sV, &tmap_kv, bar, (2 * nh + head0) * DH, c0, r0 + j * NA_BLK_ROWS, b);
      }
    }
    return;
  }

  // ---------------------------------------------------- warpgroup: S = Q K^T (wgmma) -> softmax, thread = row -> O += P V (wgmma)
  const int row = warp * 32 + lane;
  float m = -INFINITY, l = 0.f;
  // this row's query and the origin of its clamped 7x7 window
  const int na_qi = qi0 + (row >> 4), na_qj = qj0 + (row & 15);
  const int na_rs = min(max(na_qi - 3, 0), p.h - 7), na_cs = min(max(na_qj - 3, 0), p.w - 7);
  auto key_ok = [&](int j, int t) -> bool {      // is tile column t of key block j inside this row's neighbourhood?
    const int dr = (t * 745) >> 14;               // t / 22 for t < 128
    const int kr = r0 + j * NA_BLK_ROWS + dr, kc = c0 + (t - dr * NA_KW);
    return t < NA_BLK_KEYS && (unsigned)(kr - na_rs) < 7u && (unsigned)(kc - na_cs) < 7u;
  };
  const uint32_t q_addr = tc::smem_u32(sQ), k_addr = tc::smem_u32(sK), p_addr = tc::smem_u32(sP);
  const uint64_t vdesc = tc::smem_desc_mn_sw128(tc::smem_u32(sV), 1024, 1024);
  float o0[32], o1[32];                        // O rows 0-63 / 64-127, accumulated over the key blocks of the P V pass
#pragma unroll
  for (int i = 0; i < 32; ++i) o0[i] = o1[i] = 0.f;
  tc::mbar_wait_nocall(&bars->q, 0);
  for (int it = 0; it < n_iter; ++it) {
    const int j = it % nblk;
    const int pass = (two_pass && it < nblk) ? 0 : 1;
    bars->kv.wait(PipeState<1>::at(it));
    // S = Q K^T, one M = 64 half at a time -> fp32 tile
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float s[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) s[i] = 0.f;
      const uint64_t qd = tc::smem_desc_k_sw128(q_addr + (uint32_t)h * 8192u), kd = tc::smem_desc_k_sw128(k_addr);
      tc::wg_fence_acc(s);
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k) tc::wgmma_128(s, qd + 2ull * k, kd + 2ull * k, 1u);
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(s);
      tc::acc_store(sS, S_LD, 64 * h, s);
    }
    tc::named_barrier_sync(tc::BAR_WG, 128);            // S complete; every read of Q and K is done
    if (pass == 0) {
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        float v[32];
        tc::acc_ld32(sS, S_LD, row, c * 32, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) m = fmaxf(m, key_ok(j, c * 32 + i) ? v[i] : -INFINITY);
      }
    } else {
      if constexpr (bounded) m = __ldg(p.bound + head0);
      if (!two_pass && !bounded) {             // single block: the row maximum comes from this very tile
        float mm = -INFINITY;
#pragma unroll 1
        for (int c2 = 0; c2 < 4; ++c2) {
          float u[32];
          tc::acc_ld32(sS, S_LD, row, c2 * 32, u);
#pragma unroll
          for (int i = 0; i < 32; ++i) mm = fmaxf(mm, u[i]);
        }
        m = mm;
      }
      const float mb = m * LOG2E;
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        float v[32];
        tc::acc_ld32(sS, S_LD, row, c * 32, v);
        uint32_t pk[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float p0 = key_ok(j, c * 32 + 2 * i) ? exp2f(fmaf(v[2 * i], LOG2E, -mb)) : 0.f;
          const float p1 = key_ok(j, c * 32 + 2 * i + 1) ? exp2f(fmaf(v[2 * i + 1], LOG2E, -mb)) : 0.f;
          pk[i] = tc::pack_bf16x2(p0, p1);
          float q0, q1;
          tc::unpack_bf16x2(pk[i], q0, q1);     // l accumulates exactly what the P V MMA sees
          l += q0 + q1;
        }
        uint8_t* pt = sP + (c >> 1) * TILE_BYTES;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          *reinterpret_cast<uint4*>(pt + tc::sw128_offset(row, (c & 1) * 4 + jj)) = make_uint4(pk[jj * 4], pk[jj * 4 + 1], pk[jj * 4 + 2], pk[jj * 4 + 3]);
      }
    }
    if (pass == 1) {
      tc::fence_proxy_async();                 // P (generic-proxy writes) -> visible to the tensor core
      tc::named_barrier_sync(tc::BAR_WG, 128);
      tc::wg_fence_acc(o0);
      tc::wg_fence_acc(o1);
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < ROWS / 16; ++k) {    // 16 keys per step: K-block k / 4 of P, rows 16 k.. of V (two 8-row groups)
        const uint32_t pa = p_addr + (uint32_t)((k >> 2) * TILE_BYTES);
        const uint64_t bd = vdesc + (uint64_t)(k * ((16 * 128) >> 4));
        tc::wgmma_64<1>(o0, tc::smem_desc_k_sw128(pa) + 2ull * (k & 3), bd, 1u);
        tc::wgmma_64<1>(o1, tc::smem_desc_k_sw128(pa + 8192u) + 2ull * (k & 3), bd, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(o0);
      tc::wg_fence_acc(o1);
    }
    tc::named_barrier_sync(tc::BAR_WG, 128);            // S, K, V and P are free for the next key block
    if (lane == 0 && it + 1 < n_iter) bars->kv.release(PipeState<1>::at(it));   // none after the last block: its phase is never waited for
  }
  // ------------------------------------------------------ O / l -> out
  tc::acc_store(sS, S_LD, 0, o0);
  tc::acc_store(sS, S_LD, 64, o1);
  tc::named_barrier_sync(tc::BAR_WG, 128);
  const float inv = 1.f / l;
  const int64_t token = (int64_t)na_qi * p.w + na_qj;
  uint4* dst = reinterpret_cast<uint4*>(p.out + (((int64_t)b * p.h * p.w + token) * nh + head0) * DH);
#pragma unroll 1
  for (int c = 0; c < 2; ++c) {
    float v[32];
    tc::acc_ld32(sS, S_LD, row, c * 32, v);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
      dst[c * 4 + jj] = make_uint4(tc::pack_bf16x2(v[jj * 8 + 0] * inv, v[jj * 8 + 1] * inv), tc::pack_bf16x2(v[jj * 8 + 2] * inv, v[jj * 8 + 3] * inv),
                                   tc::pack_bf16x2(v[jj * 8 + 4] * inv, v[jj * 8 + 5] * inv), tc::pack_bf16x2(v[jj * 8 + 6] * inv, v[jj * 8 + 7] * inv));
  }
}

constexpr size_t ATTN_NA_SMEM = 5 * TILE_BYTES + (size_t)ROWS * S_LD * 4 + 1024 + 128;

}  // namespace

static bool g_attn_tc_disabled = [] {
  const char* e = getenv("KDB200_DISABLE_TC_ATTN");
  const char* f = getenv("KDB200_DISABLE_TC");
  return (e != nullptr && e[0] == '1') || (f != nullptr && f[0] == '1');
}();

bool tc_attention_supported(int h, int w, int nh, int e, int attn_type, int attn_param) {
  if (g_attn_tc_disabled || e != 64) return false;
  if (attn_type == KDB_ATTN_SHIFTED_WINDOW) return attn_param == 8 && h % 8 == 0 && w % 8 == 0 && nh % 2 == 0;
  if (attn_type == KDB_ATTN_GLOBAL) return (h * w) % 128 == 0 && (h * w) / 128 <= 64;
  if (attn_type == KDB_ATTN_NEIGHBORHOOD) return attn_param == 7 && h % NA_QH == 0 && w % NA_QW == 0 && h >= NA_KH && w >= NA_KW;
  return false;
}

// persistent WINDOW / GLOBAL launch; programmatic dependent launch, so that barrier init overlaps the tail of the qkv projection
template <int MODE>
static int launch_ws(cudaStream_t st, const CUtensorMap& tin, const CUtensorMap& tout, const AttnParams& p) {
  const bool bounded = p.bound != nullptr;
  auto kernel = bounded ? attn_ws_kernel<MODE, true> : attn_ws_kernel<MODE, false>;
  static bool opened[2] = {false, false};
  if (int rc = set_smem_once(kernel, opened[bounded], (int)WS_SMEM)) return rc;
  KDB_CUDA(launch_pdl(kernel, persistent_grid(p.n_tiles), dim3(WS_THREADS), WS_SMEM, st, tin, tout, p));
  return 0;
}

int launch_attention_tc(const bf16* qkv, bf16* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                        cudaStream_t st, const float* logit_bound) {
  KDB_REQUIRE(tc_attention_supported(h, w, nh, e, attn_type, attn_param), KDB_ERR_UNSUPPORTED, "attention_tc: unsupported shape");
  KDB_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, KDB_ERR_BAD_ARG,
              "attention_tc: operands must be 16-byte aligned");
  const uint64_t F = 3ull * nh * e, C = (uint64_t)nh * e;
  AttnParams p{};
  p.out = out;
  p.B = B; p.h = h; p.w = w; p.nh = nh; p.shift = shift;
  p.bound = logit_bound;
  CUtensorMap tm, to;
  int rc;
  if (attn_type == KDB_ATTN_SHIFTED_WINDOW) {
    KDB_REQUIRE(shift == 0 || shift == 4, KDB_ERR_UNSUPPORTED, "attention_tc: window shift must be 0 or window/2");
    if ((rc = make_tmap_tokens(&tm, qkv, F, B, h, w, DH, 4, 4))) return rc;     // one quadrant of a window
    if ((rc = make_tmap_tokens(&to, out, C, B, h, w, DH, 4, 4))) return rc;
    p.nblk = 1;
    p.n_tiles = B * (h / 8) * (w / 8) * (nh / 2);
    if ((rc = launch_ws<MODE_WINDOW>(st, tm, to, p))) return rc;
  } else if (attn_type == KDB_ATTN_NEIGHBORHOOD) {
    CUtensorMap tkv;
    if ((rc = make_tmap_tokens(&tm, qkv, F, B, h, w, DH, NA_QW, NA_QH))) return rc;
    if ((rc = make_tmap_tokens(&tkv, qkv, F, B, h, w, DH, NA_KW, NA_BLK_ROWS))) return rc;
    const bool bounded = p.bound != nullptr;
    auto kernel = bounded ? attn_na_kernel<true> : attn_na_kernel<false>;
    static bool opened[2] = {false, false};
    if ((rc = set_smem_once(kernel, opened[bounded], (int)ATTN_NA_SMEM))) return rc;
    p.nblk = 3;      // 14 halo rows = 5 + 5 + 4
    dim3 grid((unsigned)((h / NA_QH) * (w / NA_QW)), (unsigned)nh, (unsigned)B);
    KDB_CUDA(launch_pdl(kernel, grid, dim3(160), ATTN_NA_SMEM, st, tm, tkv, p));
  } else {
    const uint64_t T = (uint64_t)h * w;
    const uint64_t dims[3] = {F, T, (uint64_t)B}, dims_o[3] = {C, T, (uint64_t)B};
    const uint64_t strides[2] = {F * 2, F * 2 * T}, strides_o[2] = {C * 2, C * 2 * T};
    const uint32_t box[3] = {DH, ROWS, 1}, box_o[3] = {DH, 64, 1};
    if ((rc = make_tmap_bf16(&tm, qkv, 3, dims, strides, box))) return rc;
    if ((rc = make_tmap_bf16(&to, out, 3, dims_o, strides_o, box_o))) return rc;
    p.nblk = (int)(T / ROWS);
    p.n_tiles = B * nh * p.nblk;
    if ((rc = launch_ws<MODE_GLOBAL>(st, tm, to, p))) return rc;
  }
  KDB_LAUNCH_CHECK(F_ATTN_TC, st);
  return 0;
}

}  // namespace kdb
