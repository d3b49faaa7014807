// tc_attention.cu -- bf16 attention on the sm_90a tensor core (wgmma) for the attention types of the model configurations:
//   * shifted-window attention, 8x8 windows, d_head 64 (reference image_transformer_v2.py:253-337,446-476)
//   * global attention, sequence a multiple of 128, d_head 64 (:355-396)
// q and k arrive already cosine-normalised and rotated (qknorm_rope kernel); softmax scale is 1.0.
//
// One CTA = one 128-row S tile:
//   WINDOW : rows = 2 heads x 64 tokens of one window; S = [Q_h0;Q_h1][K_h0;K_h1]^T is computed as one 128x128
//            MMA and only the two 64x64 diagonal blocks are used (attention is ~2 % of the model's MACs: the
//            wasted half is cheaper than half-rate M=64 MMAs).  The roll (:274) is pure index arithmetic: the window
//            is fetched as four 4x4-token TMA boxes (quadrants), which are exactly the seam-mask regions (:300-315).
//   GLOBAL : rows = 128 queries of one head; keys streamed in blocks of 128; exact two-pass softmax
//            (pass A: row maxima, pass B: exp / P V) so no accumulator rescaling is needed.
//   NA     : 7x7 neighbourhood attention (reference :399-443 via natten; NATTEN definition: window clamped inward at the
//            borders, always 49 keys).  Rows = an 8x16 query block of one head; its keys all lie in the clamped 14x22 halo,
//            streamed as three TMA boxes of 5 halo rows (110 keys per 128-row tile, the tail rows are masked / zero);
//            the per-query 7x7 window is a mask on S.  Same two-pass softmax as GLOBAL.
// Roles: warp 4 = TMA producer, warps 0-3 = the warpgroup that issues the MMAs and runs the softmax.  Per key block: TMA
// (SWIZZLE_128B) -> S = Q K^T (wgmma, two M = 64 halves) -> fp32 S tile in shared memory -> softmax (one thread per row) ->
// P (bf16) written to shared memory in the K-major SW128 layout -> O += P V (V consumed as an MN-major operand straight from
// the TMA tile, O in registers across key blocks) -> fp32 O tile, 1/l scaling, store.
#include "tc_common.cuh"
#include "tc_kernels.cuh"

namespace kdb {
namespace {

constexpr int ROWS = 128, DH = 64;
constexpr int TILE_BYTES = ROWS * DH * 2;    // 16 KiB: 128 rows x 128 B
constexpr float LOG2E = 1.4426950408889634f;
constexpr int S_LD = ROWS + 4;               // row pitch (floats) of the fp32 S / O tile

enum { MODE_WINDOW = 0, MODE_GLOBAL = 1, MODE_NA = 2 };

constexpr int NA_QH = 8, NA_QW = 16;          // query block of one CTA (128 queries of one head)
constexpr int NA_KH = 14, NA_KW = 22;         // its clamped key halo for a 7x7 neighbourhood
constexpr int NA_BLK_ROWS = 5;                // halo rows per key block: 5 x 22 = 110 keys (of a 128-row tile)
constexpr int NA_BLK_KEYS = NA_BLK_ROWS * NA_KW;

struct AttnParams {
  bf16* out;
  // [nh] or nullptr: upper bound of |q . k| per head.  q and k are cosine-normalised (|q| = |k| = sqrt(scale_h), reference
  // :106-114, RoPE is a rotation), so the layer's scale IS that bound and softmax can use it as a FIXED shift: exp(s - bound)
  // needs no row maximum -> GLOBAL / NA run ONE pass over the key blocks instead of two, WINDOW skips its max scan.
  const float* bound;
  int B, h, w, nh, shift, nblk;
};

struct Bars {
  uint64_t q, kv, kv_free;
};

__device__ __forceinline__ uint32_t p_offset(int row, int chunk16) {   // byte offset of 16-byte chunk `chunk16` (0..7) of `row` in a K-major SW128 tile
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk16 ^ (row & 7)) << 4));
}

template <int MODE, bool BOUNDED>
__global__ void __launch_bounds__(160, 1) attn_tc_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_kv,
                                                         const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = base;
  uint8_t* sK = base + TILE_BYTES;
  uint8_t* sV = base + 2 * TILE_BYTES;
  // P (two K-blocks of 64 keys, 32 KiB).  WINDOW has a single key block: Q and K are dead once S = Q K^T has completed, so
  // P overwrites them; GLOBAL re-uses Q for every key block and keeps P separate.
  uint8_t* sP = (MODE == MODE_WINDOW) ? sQ : base + 3 * TILE_BYTES;
  float* sS = reinterpret_cast<float*>(base + (MODE == MODE_WINDOW ? 3 : 5) * TILE_BYTES);   // fp32 S (then O) tile, row pitch S_LD
  Bars* bars = reinterpret_cast<Bars*>(sS + ROWS * S_LD);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nh = p.nh;
  // work decomposition
  int b = blockIdx.z, head0, wi = 0, wj = 0, mtile = 0;
  if constexpr (MODE == MODE_WINDOW) {
    const int nww = p.w / 8;
    wi = blockIdx.x / nww;
    wj = blockIdx.x - wi * nww;
    head0 = blockIdx.y * 2;
  } else {
    mtile = blockIdx.x;
    head0 = blockIdx.y;
  }
  int qi0 = 0, qj0 = 0, r0 = 0, c0 = 0;      // NA: query block origin and clamped halo origin
  if constexpr (MODE == MODE_NA) {
    const int nbw = p.w / NA_QW;
    qi0 = (blockIdx.x / nbw) * NA_QH;
    qj0 = (blockIdx.x % nbw) * NA_QW;
    r0 = min(max(qi0 - 3, 0), p.h - NA_KH);
    c0 = min(max(qj0 - 3, 0), p.w - NA_KW);
  }
  const int nblk = (MODE == MODE_WINDOW) ? 1 : p.nblk;
  constexpr bool bounded = BOUNDED;
  const bool two_pass = nblk > 1 && !bounded;
  const int n_iter = two_pass ? 2 * nblk : nblk;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmap);
    tc::mbar_init(&bars->q, 1);
    tc::mbar_init(&bars->kv, 1);
    tc::mbar_init(&bars->kv_free, 4);          // lane 0 of each warp of the warpgroup
    tc::fence_barrier_init();
  }
  if constexpr (MODE == MODE_NA) {   // rows 110..127 of the V tile are never written by TMA: they must be finite (P there is exactly 0)
    for (int i = threadIdx.x; i < (ROWS - NA_BLK_KEYS) * 8; i += blockDim.x)
      *reinterpret_cast<uint4*>(sV + NA_BLK_KEYS * 128 + i * 16) = make_uint4(0u, 0u, 0u, 0u);
    tc::fence_proxy_async();
  }
  __syncthreads();
  tc::pdl_wait();                              // programmatic launch: the qkv projection before us must be complete from here on
  tc::pdl_launch_dependents();

  if (warp == 4) {
    if (tc::elect_one()) {
      // ------------------------------------------------ loads of Q and of each key block (K, and V in the P V pass)
      auto load_window_tile = [&](uint8_t* dst, int t, uint64_t* bar) {
        if (p.shift == 0) {   // unshifted window: one 8x8 box per head, rows in (lr, lc) order (tensor map box = 64 x 8 x 8)
#pragma unroll
          for (int hd = 0; hd < 2; ++hd) tc::tma_load_4d(dst + hd * 64 * 128, &tmap, bar, (t * nh + head0 + hd) * DH, wj * 8, wi * 8, b);
          return;
        }
#pragma unroll
        for (int hd = 0; hd < 2; ++hd)
#pragma unroll
          for (int quad = 0; quad < 4; ++quad) {
            const int r0 = (wi * 8 + (quad >> 1) * 4 - p.shift + p.h) % p.h;   // rolled -> original coordinates (:274)
            const int c0 = (wj * 8 + (quad & 1) * 4 - p.shift + p.w) % p.w;
            tc::tma_load_4d(dst + (hd * 64 + quad * 16) * 128, &tmap, bar, (t * nh + head0 + hd) * DH, c0, r0, b);
          }
      };
      tc::mbar_arrive_expect_tx(&bars->q, TILE_BYTES);
      if constexpr (MODE == MODE_WINDOW)
        load_window_tile(sQ, 0, &bars->q);
      else if constexpr (MODE == MODE_NA)
        tc::tma_load_4d(sQ, &tmap, &bars->q, head0 * DH, qj0, qi0, b);
      else
        tc::tma_load_3d(sQ, &tmap, &bars->q, head0 * DH, mtile * ROWS, b);
      for (int it = 0; it < n_iter; ++it) {
        const int j = it % nblk;
        const bool with_v = !two_pass || it >= nblk;
        if (it > 0) tc::mbar_wait(&bars->kv_free, (uint32_t)(it - 1) & 1u);
        constexpr uint32_t KV_BYTES = (MODE == MODE_NA) ? NA_BLK_KEYS * 128 : TILE_BYTES;
        tc::mbar_arrive_expect_tx(&bars->kv, with_v ? 2 * KV_BYTES : KV_BYTES);
        if constexpr (MODE == MODE_WINDOW) {
          load_window_tile(sK, 1, &bars->kv);
          load_window_tile(sV, 2, &bars->kv);
        } else if constexpr (MODE == MODE_NA) {
          tc::tma_load_4d(sK, &tmap_kv, &bars->kv, (nh + head0) * DH, c0, r0 + j * NA_BLK_ROWS, b);
          if (with_v) tc::tma_load_4d(sV, &tmap_kv, &bars->kv, (2 * nh + head0) * DH, c0, r0 + j * NA_BLK_ROWS, b);
        } else {
          tc::tma_load_3d(sK, &tmap, &bars->kv, (nh + head0) * DH, j * ROWS, b);
          if (with_v) tc::tma_load_3d(sV, &tmap, &bars->kv, (2 * nh + head0) * DH, j * ROWS, b);
        }
      }
    }
    return;
  }

  // ---------------------------------------------------- warpgroup: S = Q K^T (wgmma) -> softmax, thread = row -> O += P V (wgmma)
  const int row = warp * 32 + lane;
  float m = -INFINITY, l = 0.f;
  // window geometry of this row
  const int hd = row >> 6, quad = (row & 63) >> 4;
  const bool seam_r = MODE == MODE_WINDOW && p.shift > 0 && wi == 0;
  const bool seam_c = MODE == MODE_WINDOW && p.shift > 0 && wj == 0;
  // NA: this row's query and the origin of its clamped 7x7 window
  const int na_qi = qi0 + (row >> 4), na_qj = qj0 + (row & 15);
  const int na_rs = min(max(na_qi - 3, 0), p.h - 7), na_cs = min(max(na_qj - 3, 0), p.w - 7);
  auto key_ok = [&](int j, int t) -> bool {      // is tile column t of key block j inside this row's neighbourhood?
    if constexpr (MODE != MODE_NA) return true;
    const int dr = (t * 745) >> 14;               // t / 22 for t < 128
    const int kr = r0 + j * NA_BLK_ROWS + dr, kc = c0 + (t - dr * NA_KW);
    return t < NA_BLK_KEYS && (unsigned)(kr - na_rs) < 7u && (unsigned)(kc - na_cs) < 7u;
  };
  const uint32_t q_addr = tc::smem_u32(sQ), k_addr = tc::smem_u32(sK), p_addr = tc::smem_u32(sP);
  const uint64_t vdesc = tc::smem_desc_mn_sw128(tc::smem_u32(sV), 1024, 1024);
  float o0[32], o1[32];                        // O rows 0-63 / 64-127, accumulated over the key blocks of the P V pass
#pragma unroll
  for (int i = 0; i < 32; ++i) o0[i] = o1[i] = 0.f;
  tc::mbar_wait(&bars->q, 0);
  for (int it = 0; it < n_iter; ++it) {
    const int j = it % nblk;
    const int pass = (two_pass && it < nblk) ? 0 : 1;
    tc::mbar_wait(&bars->kv, (uint32_t)it & 1u);
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
    tc::named_barrier_sync(1, 128);            // S complete; every read of Q and K is done (WINDOW: P may overwrite them)
    if (pass == 0) {
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        float v[32];
        tc::acc_ld32(sS, S_LD, row, c * 32, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) m = fmaxf(m, key_ok(j, c * 32 + i) ? v[i] : -INFINITY);
      }
    } else if constexpr (MODE != MODE_WINDOW) {
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
          *reinterpret_cast<uint4*>(pt + p_offset(row, (c & 1) * 4 + jj)) = make_uint4(pk[jj * 4], pk[jj * 4 + 1], pk[jj * 4 + 2], pk[jj * 4 + 3]);
      }
    } else {
      // WINDOW: own head's 64 key columns live at [64*hd, 64*hd+64); the other head's block is garbage -> zeros in P
      float v[64];
      {
        float t0[32], t1[32];
        tc::acc_ld32(sS, S_LD, row, hd * 64, t0);
        tc::acc_ld32(sS, S_LD, row, hd * 64 + 32, t1);
#pragma unroll
        for (int i = 0; i < 32; ++i) { v[i] = t0[i]; v[32 + i] = t1[i]; }
      }
      if constexpr (!bounded) {
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int kq = i >> 4;
          const bool ok = (!seam_r || ((kq >> 1) == (quad >> 1))) && (!seam_c || ((kq & 1) == (quad & 1)));
          v[i] = ok ? v[i] : -INFINITY;
          m = fmaxf(m, v[i]);
        }
      } else {
        m = __ldg(p.bound + head0 + hd);          // fixed shift: no maximum scan; masked keys get p = 0 below
      }
      const float mb = m * LOG2E;
      uint8_t* own = sP + hd * TILE_BYTES;
      uint8_t* other = sP + (1 - hd) * TILE_BYTES;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        uint32_t pk[4];
        bool ok = true;                        // (bounded) seam mask of this 8-key group: zero probability instead of -inf logit
        if constexpr (bounded) {
          const int kq = jj >> 1;
          ok = (!seam_r || ((kq >> 1) == (quad >> 1))) && (!seam_c || ((kq & 1) == (quad & 1)));
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float p0 = exp2f(fmaf(v[jj * 8 + 2 * t], LOG2E, -mb)), p1 = exp2f(fmaf(v[jj * 8 + 2 * t + 1], LOG2E, -mb));
          if constexpr (bounded) {
            p0 = ok ? p0 : 0.f;
            p1 = ok ? p1 : 0.f;
          }
          pk[t] = tc::pack_bf16x2(p0, p1);
          float q0, q1;
          tc::unpack_bf16x2(pk[t], q0, q1);
          l += q0 + q1;
        }
        *reinterpret_cast<uint4*>(own + p_offset(row, jj)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        *reinterpret_cast<uint4*>(other + p_offset(row, jj)) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    if (pass == 1) {
      tc::fence_proxy_async();                 // P (generic-proxy writes) -> visible to the tensor core
      tc::named_barrier_sync(1, 128);
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
    tc::named_barrier_sync(1, 128);            // S, K, V and P are free for the next key block
    if (lane == 0 && it + 1 < n_iter) tc::mbar_arrive(&bars->kv_free);
  }
  // ------------------------------------------------------ O / l -> out
  tc::acc_store(sS, S_LD, 0, o0);
  tc::acc_store(sS, S_LD, 64, o1);
  tc::named_barrier_sync(1, 128);
  const float inv = 1.f / l;
  int64_t token;
  int head;
  if constexpr (MODE == MODE_WINDOW) {
    int oi, oj;
    if (p.shift == 0) {
      oi = wi * 8 + ((row & 63) >> 3);
      oj = wj * 8 + (row & 7);
    } else {
      const int lr = (row & 15) >> 2, lc = row & 3;
      oi = (wi * 8 + (quad >> 1) * 4 + lr - p.shift + p.h) % p.h;
      oj = (wj * 8 + (quad & 1) * 4 + lc - p.shift + p.w) % p.w;
    }
    token = (int64_t)oi * p.w + oj;
    head = head0 + hd;
  } else if constexpr (MODE == MODE_NA) {
    token = (int64_t)na_qi * p.w + na_qj;
    head = head0;
  } else {
    token = (int64_t)mtile * ROWS + row;
    head = head0;
  }
  uint4* dst = reinterpret_cast<uint4*>(p.out + (((int64_t)b * p.h * p.w + token) * nh + head) * DH);
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


constexpr size_t ATTN_S_BYTES = (size_t)ROWS * S_LD * 4;
constexpr size_t ATTN_SMEM = 5 * TILE_BYTES + ATTN_S_BYTES + 1024 + 128;          // GLOBAL, NA
constexpr size_t ATTN_SMEM_WINDOW = 3 * TILE_BYTES + ATTN_S_BYTES + 1024 + 128;   // WINDOW (P aliases Q,K)

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

// programmatic dependent launch: barrier init overlaps the tail of the qkv projection (KDB200_NO_PDL=1 disables)
template <int MODE>
static cudaError_t set_attn_smem(size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel<MODE, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(attn_tc_kernel<MODE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

template <int MODE>
static cudaError_t launch_attn(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tkv, const AttnParams& p) {
  static const bool no_pdl = [] {
    const char* e = getenv("KDB200_NO_PDL");
    return e != nullptr && e[0] == '1';
  }();
  cudaLaunchConfig_t lc{};
  lc.gridDim = grid;
  lc.blockDim = dim3(160);
  lc.dynamicSmemBytes = smem;
  lc.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = attr;
  lc.numAttrs = no_pdl ? 0 : 1;
  if (p.bound != nullptr) return cudaLaunchKernelEx(&lc, attn_tc_kernel<MODE, true>, tq, tkv, p);
  return cudaLaunchKernelEx(&lc, attn_tc_kernel<MODE, false>, tq, tkv, p);
}

int launch_attention_tc(const bf16* qkv, bf16* out, int B, int h, int w, int nh, int e, int attn_type, int attn_param, int shift,
                        cudaStream_t st, const float* logit_bound) {
  KDB_REQUIRE(tc_attention_supported(h, w, nh, e, attn_type, attn_param), KDB_ERR_UNSUPPORTED, "attention_tc: unsupported shape");
  KDB_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, KDB_ERR_BAD_ARG,
              "attention_tc: operands must be 16-byte aligned");
  const uint64_t F = 3ull * nh * e;
  AttnParams p{};
  p.out = out;
  p.B = B; p.h = h; p.w = w; p.nh = nh; p.shift = shift;
  p.bound = logit_bound;
  CUtensorMap tm;
  static bool attr_w = false, attr_g = false;
  if (attn_type == KDB_ATTN_SHIFTED_WINDOW) {
    KDB_REQUIRE(shift == 0 || shift == 4, KDB_ERR_UNSUPPORTED, "attention_tc: window shift must be 0 or window/2");
    const uint64_t dims[4] = {F, (uint64_t)w, (uint64_t)h, (uint64_t)B};
    const uint64_t strides[3] = {F * 2, F * 2 * w, F * 2 * w * h};
    const uint32_t box_q[4] = {DH, 4, 4, 1}, box_f[4] = {DH, 8, 8, 1};
    int rc = make_tmap_bf16(&tm, qkv, 4, dims, strides, shift == 0 ? box_f : box_q);
    if (rc) return rc;
    if (!attr_w) {
      KDB_CUDA(set_attn_smem<MODE_WINDOW>(ATTN_SMEM_WINDOW));
      attr_w = true;
    }
    p.nblk = 1;
    dim3 grid((unsigned)((h / 8) * (w / 8)), (unsigned)(nh / 2), (unsigned)B);
    KDB_CUDA(launch_attn<MODE_WINDOW>(grid, ATTN_SMEM_WINDOW, st, tm, tm, p));
  } else if (attn_type == KDB_ATTN_NEIGHBORHOOD) {
    static bool attr_n = false;
    CUtensorMap tkv;
    const uint64_t dims[4] = {F, (uint64_t)w, (uint64_t)h, (uint64_t)B};
    const uint64_t strides[3] = {F * 2, F * 2 * w, F * 2 * w * h};
    const uint32_t box_q[4] = {DH, NA_QW, NA_QH, 1}, box_kv[4] = {DH, NA_KW, NA_BLK_ROWS, 1};
    int rc = make_tmap_bf16(&tm, qkv, 4, dims, strides, box_q);
    if (rc) return rc;
    if ((rc = make_tmap_bf16(&tkv, qkv, 4, dims, strides, box_kv))) return rc;
    if (!attr_n) {
      KDB_CUDA(set_attn_smem<MODE_NA>(ATTN_SMEM));
      attr_n = true;
    }
    p.nblk = 3;      // 14 halo rows = 5 + 5 + 4
    dim3 grid((unsigned)((h / NA_QH) * (w / NA_QW)), (unsigned)nh, (unsigned)B);
    KDB_CUDA(launch_attn<MODE_NA>(grid, ATTN_SMEM, st, tm, tkv, p));
  } else {
    const uint64_t T = (uint64_t)h * w;
    const uint64_t dims[3] = {F, T, (uint64_t)B};
    const uint64_t strides[2] = {F * 2, F * 2 * T};
    const uint32_t box[3] = {DH, ROWS, 1};
    int rc = make_tmap_bf16(&tm, qkv, 3, dims, strides, box);
    if (rc) return rc;
    if (!attr_g) {
      KDB_CUDA(set_attn_smem<MODE_GLOBAL>(ATTN_SMEM));
      attr_g = true;
    }
    p.nblk = (int)(T / ROWS);
    dim3 grid((unsigned)(T / ROWS), (unsigned)nh, (unsigned)B);
    KDB_CUDA(launch_attn<MODE_GLOBAL>(grid, ATTN_SMEM, st, tm, tm, p));
  }
  KDB_LAUNCH_CHECK(F_ATTN_TC, st);
  return 0;
}

}  // namespace kdb
