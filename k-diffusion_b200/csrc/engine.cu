// engine.cu -- host-side execution plan for the image_transformer_v2 denoiser
// (reference: k_diffusion/models/image_transformer_v2.py:667-762 and layers.py:88-90), and for image_transformer_v1
// (image_transformer_v1.py:280-344), which runs as a one-level model with global attention through weights derived at finalize.
//
// The engine owns no activations: the caller passes one workspace; the plan carves it.  Weights are
// borrowed device pointers keyed by the reference state-dict names; kdb_model_finalize builds the
// derived tables (bf16 copies, concatenated AdaRMSNorm projection, position grids, the QkRope tables).
#include <algorithm>
#include <cmath>
#include <map>
#include <string>
#include <type_traits>
#include <vector>

#include "model_core.cuh"
#include "unet_kernels.cuh"
#include "tc_kernels.cuh"

namespace kdb {

// The tf32 training precision's copies of a token-stream weight [N, K] (ensure_tf32): w rounded to the nearest tf32 (ties away from
// zero), the forward's B operand, and t = its transpose [K, N] rounded alike, the input gradient's
struct Tf32W {
  float* w = nullptr;
  float* t = nullptr;
};

// A token-stream Linear (qkv, out, up, down, merge, split): its fp32 weight w [N, K] and the weight's copy for each route, wb for bf16
// sampling (bind, at finalize) and t for tf32 training (ensure_tf32).  lin_fwd, lin_dx and lin_dw pick the copy and the kernel.
struct Lin {
  const float* w = nullptr;
  bf16* wb = nullptr;
  Tf32W t;
  int N = 0, K = 0;
};

struct LayerPlan {
  std::string prefix;
  int level = 0, attn_type = 0, attn_param = 0, shift = 0;
  int C = 0, dff = 0, nh = 0, e = 0;
  int ada_attn = -1, ada_ff = -1;   // offsets into a conditioning row
  const float *attn_norm_w = nullptr, *ff_norm_w = nullptr;
  Lin qkv, out, up, down;
  QkRope qr;                         // cosine-sim + RoPE of q and k (freqs always, scale for v1: finalize's tables)
  bf16* up_wb_il = nullptr;          // up_proj rows interleaved (value/gate) for the fused GEGLU epilogue
  bool bounded = false;              // every qr.scale[h] in (0, KDB_ATTN_MAX_BOUND]: the scale is the attention kernels' fixed softmax shift
  bf16 *qkv_wf = nullptr, *up_wf = nullptr;   // per-evaluation copies with the AdaRMSNorm channel scale folded in (fused norm)
};

struct PosTables {
  std::vector<float*> pos;          // per level: [T_l, 2] (y, x)
  std::vector<float2*> rope;        // per layer (KdbModel::layers): [T_l, nh, R/2] (cos, sin) of the RoPE angles, or nullptr
};

}  // namespace kdb

using namespace kdb;

struct KdbModel : ModelCore {
  KdbModelConfig cfg{};
  std::vector<LayerPlan> layers;   // in execution order (for_each_layer)
  std::vector<Lin> merge, split;   // per level l < n_levels - 1
  std::vector<const float*> split_fac;
  const float *patch_in_w = nullptr, *out_norm = nullptr, *patch_out_w = nullptr;
  float* ada_cat = nullptr;
  FoldDesc* fold_descs = nullptr;   // device table for launch_fold_norm_weights
  int n_fold = 0;
  bool fuse_norm = true;
  bf16* patch_out_wb = nullptr;     // patch_out.proj.weight zero-padded to 64 rows (tensor-core patch-out)
  bf16* patch_out_wf = nullptr;     // the same with out_norm.scale folded in (fused out_norm)
  bf16* patch_in_wb = nullptr;      // patch_in.proj.weight, columns permuted to (c, nh, nw) and padded to 64 (tensor-core patch-in)
  int ada_total = 0;
  CondWeights cw{};
  std::map<std::pair<int, int>, PosTables> pos_cache;   // position tables per token grid, in owned allocations
};

namespace {

int make_bf16(KdbModel* m, const float* src, int64_t n, bf16** dst, cudaStream_t st) {
  int rc = m->alloc(dst, (size_t)n);
  if (rc) return rc;
  return launch_f32_to_bf16(src, *dst, n, st);
}

// the n floats at device pointer src, on the host
int download(const float* src, size_t n, std::vector<float>& out, cudaStream_t st) {
  out.resize(n);
  KDB_CUDA(cudaMemcpyAsync(out.data(), src, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
  KDB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// a device copy of host floats, owned by the model
int upload(KdbModel* m, const std::vector<float>& v, const float** out, cudaStream_t st) {
  float* d = nullptr;
  int rc = m->alloc(&d, v.size());
  if (rc) return rc;
  KDB_CUDA(cudaMemcpyAsync(d, v.data(), sizeof(float) * v.size(), cudaMemcpyHostToDevice, st));
  KDB_CUDA(cudaStreamSynchronize(st));
  *out = d;
  return 0;
}

// an owned copy of the [rows, cols] matrix src whose row r (cols == 1: element r) is row perm(r) of src
template <typename P>
int permuted_rows(KdbModel* m, const float* src, int64_t rows, int64_t cols, P&& perm, const float** out, cudaStream_t st) {
  std::vector<float> a, b((size_t)(rows * cols));
  int rc = download(src, (size_t)(rows * cols), a, st);
  if (rc) return rc;
  for (int64_t r = 0; r < rows; ++r) std::copy_n(a.begin() + perm(r) * cols, cols, b.begin() + r * cols);
  return upload(m, b, out, st);
}

// Binds the token-stream Linear `key` [N, K]: lin.w is the state-dict tensor (with `perm`, an owned copy whose row r is its row perm(r)),
// lin.wb the bf16 copy of lin.w
template <typename P = std::nullptr_t>
int bind(KdbModel* m, Lin& lin, const std::string& key, int N, int K, cudaStream_t st, P perm = nullptr) {
  GET(key, &lin.w, N, K);
  lin.N = N;
  lin.K = K;
  if constexpr (!std::is_null_pointer_v<P>)
    if (int rc = permuted_rows(m, lin.w, N, K, perm, &lin.w, st)) return rc;
  return make_bf16(m, lin.w, (int64_t)N * K, &lin.wb, st);
}

// image_transformer_v1's patch feature order (c i j) (Patching / Unpatching, image_transformer_v1.py:223,242) -> the engine's (i j c)
// (TokenMerge / TokenSplitWithoutSkip, image_transformer_v2.py:594,607): the (c i j) index of (i j c) feature n
int64_t v1_patch_feature(int64_t n, int ch, int ph, int pw) {
  const int64_t q = n / ch, c = n - q * ch;
  return c * ph * pw + q;
}

// rows of up_proj [2F, C] reordered so that every 16-row group holds 8 value rows followed by the
// 8 matching gate rows: lets a tensor-core epilogue that owns >= 16 consecutive columns apply GEGLU.
__global__ void interleave_geglu_rows_kernel(const float* __restrict__ w, bf16* __restrict__ out, int F, int C) {
  const int64_t total = (int64_t)2 * F * C;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    const int64_t g = r / 16;
    const int j = (int)(r - g * 16);
    const int64_t src_row = (j < 8) ? (g * 8 + j) : ((int64_t)F + g * 8 + (j - 8));
    out[i] = __float2bfloat16_rn(w[src_row * C + c]);
  }
}

// dst [K, N] = src [N, K]^T rounded to the nearest tf32, ties away from zero (launch_unet_round_tf32's rounding), through 32 x 32 tiles
__global__ void __launch_bounds__(256) round_tf32_transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int K) {
  __shared__ float t[32][33];
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8)
    if (n0 + i < N && k0 + tx < K) t[i][tx] = src[(int64_t)(n0 + i) * K + k0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (k0 + i < K && n0 + tx < N) {
      uint32_t r;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(t[tx][i]));
      dst[(int64_t)(k0 + i) * N + n0 + tx] = __uint_as_float(r);
    }
}

// The layers in execution order, which is also the order of KdbModel::layers and of the conditioning row: down levels, mid, up levels
// (outermost last); level l < n-1 has depth[l] layers on the way down and as many on the way up.  f(prefix, level, index) receives
// each layer's state-dict prefix, level and index within the level, which picks the shift (image_transformer_v2.py:697: an up level's
// index continues after its down level).  Stops at the first nonzero return.
template <typename F>
int for_each_layer(const KdbModelConfig& c, F&& f) {
  const int n = c.n_levels;
  int rc = 0;
  if (c.family == KDB_FAMILY_ITV1) {   // image_transformer_v1.py:296: blocks.<i>, one level
    for (int i = 0; i < c.depth[0] && rc == 0; ++i) rc = f("blocks." + std::to_string(i) + ".", 0, i);
    return rc;
  }
  for (int l = 0; l < n - 1; ++l)
    for (int i = 0; i < c.depth[l] && rc == 0; ++i) rc = f("down_levels." + std::to_string(l) + "." + std::to_string(i) + ".", l, i);
  for (int i = 0; i < c.depth[n - 1] && rc == 0; ++i) rc = f("mid_level." + std::to_string(i) + ".", n - 1, i);
  for (int l = n - 2; l >= 0; --l)
    for (int i = 0; i < c.depth[l] && rc == 0; ++i) rc = f("up_levels." + std::to_string(l) + "." + std::to_string(i) + ".", l, i + c.depth[l]);
  return rc;
}

int plan_layer(KdbModel* m, LayerPlan& L, const std::string& prefix, int level, int index, int* ada_off, cudaStream_t st) {
  const KdbModelConfig& c = m->cfg;
  const int mw = c.mapping_width;
  L.prefix = prefix;
  L.level = level;
  L.C = c.width[level];
  L.dff = c.d_ff[level];
  L.attn_type = c.attn_type[level];
  L.attn_param = c.attn_param[level];
  if (L.attn_type != KDB_ATTN_NONE) {
    L.e = c.d_head[level];
    KDB_REQUIRE(L.e > 0 && L.C % L.e == 0, KDB_ERR_BAD_SHAPE, "level %d: width %d not divisible by d_head %d", level, L.C, L.e);
    L.nh = L.C / L.e;
    // image_transformer_v2.py:523 -- odd layer index => shift by half a window
    L.shift = (L.attn_type == KDB_ATTN_SHIFTED_WINDOW && (index % 2 == 1)) ? L.attn_param / 2 : 0;
    const std::string a = prefix + "self_attn.";
    GET(a + "norm.linear.weight", &L.attn_norm_w, L.C, mw);
    L.ada_attn = *ada_off;
    *ada_off += L.C;
    int rc;
    const int e = L.e, nh = L.nh;
    std::vector<float> hs, tab((size_t)nh * (e / 2));   // the scale per head; a QkRope frequency table wide enough for R = e
    if (c.family == KDB_FAMILY_ITV1) {
      // QKNorm + SDPA (image_transformer_v1.py:108-128,163-169): q . k exp(0.5 s - 0.25 ln e)^2 e / sqrt(mean q^2 + eps)(mean k^2 + eps) / sqrt(e)
      // = exp(s) q . k / sqrt((sum q^2 + e eps)(sum k^2 + e eps)), the cosine-sim logit with scale exp(min(s, ln 100)) (proj_'s clamp,
      // :119-123) and eps e * 1e-6.  AxialRoPE (axial_rope.py:86-107) turns the pairs (2j, 2j+1) of all e columns by pos_y exp(freqs_h[j])
      // (j < e/4) or pos_x exp(freqs_w[j - e/4]): half-split RoPE of R = e on q and k rows permuted within each head (new j <- old 2j,
      // new j + e/2 <- old 2j + 1), which changes neither q . k nor the row norms.  v keeps its rows.
      const float *s, *fh, *fw;
      GET(a + "qk_norm.scale", &s, nh);
      GET(a + "pos_emb.freqs_h", &fh, nh, e / 4);
      GET(a + "pos_emb.freqs_w", &fw, nh, e / 4);
      if ((rc = download(s, nh, hs, st))) return rc;
      for (float& v : hs) v = std::exp(std::min(v, std::log(100.f)));
      std::vector<float> y, x;
      if ((rc = download(fh, (size_t)nh * (e / 4), y, st)) || (rc = download(fw, (size_t)nh * (e / 4), x, st))) return rc;
      for (int h = 0; h < nh; ++h)
        for (int j = 0; j < e / 4; ++j) {
          tab[(size_t)h * (e / 2) + j] = std::exp(y[(size_t)h * (e / 4) + j]);
          tab[(size_t)h * (e / 2) + e / 4 + j] = std::exp(x[(size_t)h * (e / 4) + j]);
        }
      const int64_t C = L.C;
      auto perm = [C, e](int64_t r) {
        if (r >= 2 * C) return r;
        const int64_t base = r - r % e, j = r % e;
        return base + (j < e / 2 ? 2 * j : 2 * (j - e / 2) + 1);
      };
      if ((rc = bind(m, L.qkv, a + "qkv_proj.weight", 3 * L.C, L.C, st, perm)) || (rc = upload(m, hs, &L.qr.scale, st))) return rc;
      L.qr.eps = (float)e * 1e-6f;
      L.qr.R = e;
    } else {
      // image_transformer_v2.py:106-114,187-199: cosine sim with eps 1e-6, and AxialRoPE(d_head // 2) whose freqs [nh, e/8] serve both axes
      const float* f;
      GET(a + "scale", &L.qr.scale, nh);
      GET(a + "pos_emb.freqs", &f, nh, e / 8);
      std::vector<float> fv;
      if ((rc = bind(m, L.qkv, a + "qkv_proj.weight", 3 * L.C, L.C, st)) || (rc = download(L.qr.scale, nh, hs, st)) ||
          (rc = download(f, (size_t)nh * (e / 8), fv, st)))
        return rc;
      tab.resize((size_t)nh * (e / 4));
      for (int h = 0; h < nh; ++h)
        for (int j = 0; j < e / 4; ++j) tab[(size_t)h * (e / 4) + j] = fv[(size_t)h * (e / 8) + j % (e / 8)];
      L.qr.eps = 1e-6f;
      L.qr.R = e / 2;
    }
    if ((rc = upload(m, tab, &L.qr.freqs, st)) || (rc = bind(m, L.out, a + "out_proj.weight", L.C, L.C, st))) return rc;
    // |q . k| <= scale_h after the cosine-similarity normalisation: usable as a fixed softmax shift while exp(-2 scale) stays normal
    L.bounded = true;
    for (float v : hs) L.bounded = L.bounded && v > 0.f && v <= KDB_ATTN_MAX_BOUND;
    if ((rc = m->alloc(&L.qkv_wf, (size_t)3 * L.C * L.C))) return rc;
  }
  const std::string f = prefix + "ff.";
  GET(f + "norm.linear.weight", &L.ff_norm_w, L.C, mw);
  L.ada_ff = *ada_off;
  *ada_off += L.C;
  int rc;
  if ((rc = bind(m, L.up, f + "up_proj.weight", 2 * L.dff, L.C, st)) || (rc = bind(m, L.down, f + "down_proj.weight", L.C, L.dff, st))) return rc;
  if (L.dff % 8 == 0) {
    if ((rc = m->alloc(&L.up_wb_il, (size_t)2 * L.dff * L.C))) return rc;
    interleave_geglu_rows_kernel<<<kNumSMs * 4, 256, 0, st>>>(L.up.w, L.up_wb_il, L.dff, L.C);
    KDB_LAUNCH_CHECK(F_CONVERT, st);
    if ((rc = m->alloc(&L.up_wf, (size_t)2 * L.dff * L.C))) return rc;
  }
  return 0;
}

int ensure_pos(KdbModel* m, int h0, int w0, cudaStream_t st, PosTables** out) {
  const KdbModelConfig& c = m->cfg;
  auto key = std::make_pair(h0, w0);
  auto it = m->pos_cache.find(key);
  if (it != m->pos_cache.end()) {
    *out = &it->second;
    return 0;
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  KDB_CUDA(cudaStreamIsCapturing(st, &cs));
  KDB_REQUIRE(cs == cudaStreamCaptureStatusNone, KDB_ERR_UNSUPPORTED,
              "first forward for a new token grid (%dx%d) must run outside CUDA-graph capture", h0, w0);
  // axial_rope.py:31-68: cell centres in [-1,1] (short side scaled by the aspect ratio), (y, x) order.  The aspect ratio is the token
  // grid's for v2 (image_transformer_v2.py:725); v1 passes pixel_aspect_ratio = patch_h / patch_w (image_transformer_v1.py:224), which
  // makes it the image's, W / H
  const double ar = c.family == KDB_FAMILY_ITV1 ? (double)w0 * c.patch_w / ((double)h0 * c.patch_h) : (double)w0 / (double)h0;
  const double ys = ar > 1.0 ? 1.0 / ar : 1.0, xs = ar < 1.0 ? ar : 1.0;
  std::vector<double> cur((size_t)h0 * w0 * 2);
  for (int i = 0; i < h0; ++i)
    for (int j = 0; j < w0; ++j) {
      cur[((size_t)i * w0 + j) * 2 + 0] = ((2.0 * i + 1.0) / h0 - 1.0) * ys;
      cur[((size_t)i * w0 + j) * 2 + 1] = ((2.0 * j + 1.0) / w0 - 1.0) * xs;
    }
  PosTables pt;
  int h = h0, w = w0;
  for (int l = 0; l < m->cfg.n_levels; ++l) {
    std::vector<float> f(cur.begin(), cur.end());
    float* d = nullptr;
    int rc = m->alloc(&d, f.size());
    if (rc) return rc;
    KDB_CUDA(cudaMemcpyAsync(d, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    KDB_CUDA(cudaStreamSynchronize(st));
    pt.pos.push_back(d);
    if (l + 1 < m->cfg.n_levels) {   // image_transformer_v2.py:52-54: 2x2 mean
      KDB_REQUIRE(h % 2 == 0 && w % 2 == 0, KDB_ERR_BAD_SHAPE, "token grid %dx%d at level %d is not even", h, w, l);
      std::vector<double> nxt((size_t)(h / 2) * (w / 2) * 2);
      for (int i = 0; i < h / 2; ++i)
        for (int j = 0; j < w / 2; ++j)
          for (int k = 0; k < 2; ++k)
            nxt[((size_t)i * (w / 2) + j) * 2 + k] =
                0.25 * (cur[((size_t)(2 * i) * w + 2 * j) * 2 + k] + cur[((size_t)(2 * i) * w + 2 * j + 1) * 2 + k] +
                        cur[((size_t)(2 * i + 1) * w + 2 * j) * 2 + k] + cur[((size_t)(2 * i + 1) * w + 2 * j + 1) * 2 + k]);
      cur.swap(nxt);
      h /= 2;
      w /= 2;
    }
  }
  // per-layer RoPE tables (freqs are per-layer buffers of the checkpoint)
  pt.rope.assign(m->layers.size(), nullptr);
  for (size_t k = 0; k < m->layers.size(); ++k) {
    const LayerPlan& L = m->layers[k];
    if (L.attn_type == KDB_ATTN_NONE || L.e != 64) continue;
    const int T_l = (h0 >> L.level) * (w0 >> L.level);
    int rc = m->alloc(&pt.rope[k], (size_t)T_l * L.nh * (L.qr.R / 2));
    if (rc) return rc;
    if ((rc = launch_rope_table(pt.pos[L.level], L.qr.freqs, pt.rope[k], T_l, L.nh, L.qr.R / 4, st))) return rc;
  }
  KDB_CUDA(cudaStreamSynchronize(st));
  auto ins = m->pos_cache.emplace(key, std::move(pt));
  *out = &ins.first->second;
  return 0;
}

// The tf32 training precision's weight copies, built by the first tf32 call after a finalize: the Tf32W of every layer's qkv, out, up and
// down projection, then of every level's merge and split, in the model's kept allocations (w, t of each in turn)
int ensure_tf32(KdbModel* m, cudaStream_t st) {
  if (m->kept_ready) return 0;
  std::vector<Lin*> lins;
  for (LayerPlan& L : m->layers) {
    if (L.attn_type != KDB_ATTN_NONE) lins.insert(lins.end(), {&L.qkv, &L.out});
    lins.insert(lins.end(), {&L.up, &L.down});
  }
  for (int l = 0; l < m->cfg.n_levels - 1; ++l) lins.insert(lins.end(), {&m->merge[l], &m->split[l]});
  std::vector<size_t> floats;
  for (const Lin* k : lins) floats.insert(floats.end(), 2, (size_t)k->N * k->K);
  if (int rc = m->keep(floats, "tf32 training call after a finalize builds the tf32 weight copies", st)) return rc;
  for (size_t i = 0; i < lins.size(); ++i) lins[i]->t = Tf32W{m->kept[2 * i], m->kept[2 * i + 1]};
  for (const Lin* k : lins) {
    if (int rc = launch_unet_round_tf32(k->w, k->t.w, (int64_t)k->N * k->K, st)) return rc;
    round_tf32_transpose_kernel<<<dim3((unsigned)ceil_div(k->K, 32), (unsigned)ceil_div(k->N, 32)), 256, 0, st>>>(k->w, k->t.t, k->N, k->K);
    KDB_LAUNCH_CHECK(F_CONVERT, st);
  }
  m->kept_ready = true;
  return 0;
}

struct Workspace {
  std::vector<char*> xs, xup;
  char *xn = nullptr, *qkv = nullptr, *ao = nullptr, *hbuf = nullptr, *gbuf = nullptr, *mg = nullptr;
  float* rowss = nullptr;   // [tokens at level 0, SS_PARTS] sum(x^2) of the current residual stream (fused RMSNorm)
  size_t total = 0;
};

void carve(const KdbModelConfig& c, int prec, int B, int H, int W, Carver& cv, Workspace& ws) {
  const size_t s = prec == KDB_PREC_BF16 ? 2 : 4;
  const int n = c.n_levels;
  int64_t T = (int64_t)(H / c.patch_h) * (W / c.patch_w);
  size_t mx = 0, mqkv = 0, mh = 0, mg = 0;
  ws.xs.assign(n, nullptr);
  ws.xup.assign(n, nullptr);
  for (int l = 0; l < n; ++l) {
    const size_t xb = (size_t)B * T * c.width[l] * s;
    ws.xs[l] = cv.take(xb);
    if (l < n - 1) ws.xup[l] = cv.take(xb);
    mx = std::max(mx, xb);
    if (c.attn_type[l] != KDB_ATTN_NONE) mqkv = std::max(mqkv, 3 * xb);
    mh = std::max(mh, (size_t)B * T * 2 * c.d_ff[l] * s);
    if (l < n - 1) mg = std::max(mg, xb);
    T /= 4;
  }
  ws.xn = cv.take(mx);
  ws.qkv = cv.take(mqkv);
  ws.ao = cv.take(mx);
  ws.hbuf = cv.take(mh);
  ws.gbuf = cv.take(mh / 2);
  ws.mg = cv.take(mg);
  ws.rowss = cv.take<float>((size_t)B * (H / c.patch_h) * (W / c.patch_w) * SS_PARTS * sizeof(float));
  ws.total = cv.total();
}

// One forward's state: its workspace, stream and conditioning rows, and what the fused RMSNorm may use.
struct Fwd {
  int B;
  Workspace& ws;
  cudaStream_t st;
  const float* cond;
  int64_t cond_bs;          // conditioning row stride over the batch; 0: one row for every image
  const PosTables* pt;
  bool emit;                // bf16 with fused RMSNorm: producers leave the row statistics of what they write where their shape allows
  bool fold;                // emit, one shared conditioning row and a fold table: consumers take the weights with the norm scale folded in
  bool stats;               // ws.rowss holds the row statistics of the current residual stream
  bool jvp;                 // fp32 forward-mode derivative: images [B, 2B) of every token buffer carry the tangent of images [0, B)
  float* const* tape = nullptr;   // fp32 reverse mode: slot 2k / 2k+1 keep the residual stream entering layer k's attention / feed-forward half
  bool tf32 = false;              // fp32 tokens, the tf32 training route: every token-stream Linear on the tensor cores (lin_fwd, lin_dx)

  // images held by the token buffers: linear launches and taps cover them all, nonlinear primal launches the first B
  int images() const { return jvp ? 2 * B : B; }

  // a RESID / SPLIT_LERP / merge GEMM is about to write the residual stream: it leaves its row statistics if it can
  void produce(GemmEpi& e, int64_t M, int N, int K) {
    stats = emit && tc_gemm_emits_rowss(M, N, K, e);
    e.ss_out = stats ? ws.rowss : nullptr;
  }
};

// The tf32 training route's token-stream Linear: out [M, N] = A [M, K] w^T (+ resid [M, N], which may be out) with tf32 operands and fp32
// accumulation, the U-Net's 1x1 tensor-core convolution over M tokens.  w is a rounded copy: Tf32W::w for a forward Linear, Tf32W::t for
// an input gradient dA = dC W.
int linear_tf32(const float* A, const float* w, float* out, int64_t M, int N, int K, const float* resid, cudaStream_t st) {
  KDB_REQUIRE(M <= INT32_MAX, KDB_ERR_BAD_SHAPE, "tf32 linear: %lld rows", (long long)M);
  ConvArgs a;
  a.in1 = A, a.c1 = K, a.w = w, a.r1 = resid, a.rc1 = resid ? N : 0, a.out = out;
  a.B = 1, a.H = 1, a.W = (int)M, a.N = N;
  return launch_unet_conv_tf32(a, 1, st, F_GEMM_TF32);
}

// The forward of a token-stream Linear, C [M, N] = A [M, K] lin^T with the epilogue e (STORE, RESID or SPLIT_LERP): at bf16 the
// tensor-core GEMM where it runs the problem, else the SIMT GEMM, on lin.wb; at fp32 the SIMT GEMM on lin.w; on the tf32 route
// linear_tf32 on lin.t.w, which has no split epilogue: TokenSplit stores its projection to ws.mg and un-patches it with the lerp.
template <typename T>
int lin_fwd(const Fwd& f, const T* A, const Lin& lin, T* C, int64_t M, const GemmEpi& e) {
  const int N = lin.N, K = lin.K;
  if constexpr (std::is_same_v<T, bf16>) {
    if (tc_gemm_supported(M, N, K, e)) return launch_gemm_tc(A, lin.wb, C, M, N, K, e, f.st);
    return launch_gemm_simt<bf16, bf16>(A, lin.wb, C, M, N, K, e, f.st);
  } else {
    if (!f.tf32) return launch_gemm_simt<float, float>(A, lin.w, C, M, N, K, e, f.st);
    if (e.mode != EPI_SPLIT_LERP)
      return linear_tf32(A, lin.t.w, C, M, N, K, e.mode == EPI_RESID ? static_cast<const float*>(e.resid) : nullptr, f.st);
    float* y = reinterpret_cast<float*>(f.ws.mg);
    int rc = linear_tf32(A, lin.t.w, y, M, N, K, nullptr, f.st);
    return rc ? rc : launch_split_unpatch_lerp(y, static_cast<const float*>(e.resid), e.fac, C, f.images(), 2 * e.hc, 2 * e.wc, e.C, f.st);
  }
}

// The input gradient of a token-stream Linear, dA [M, K] = dC [M, N] lin: exact fp32 (gemm_vjp on lin.w), or linear_tf32 on the
// transposed copy lin.t.t on the tf32 route.  hc > 0: the Linear is a TokenMerge over an hc x wc coarse grid, and dA is un-patched 2x2 and
// added to out, the fine stream's gradient; on the tf32 route dA goes to ws.mg and a scatter kernel adds it.
int lin_dx(const Fwd& f, const float* dC, const Lin& lin, float* out, int64_t M, int hc = 0, int wc = 0) {
  const int N = lin.N, K = lin.K;
  if (!f.tf32) return launch_gemm_vjp(dC, lin.w, out, M, N, K, hc > 0 ? VJP_UNPATCH_ACC : VJP_STORE, hc, wc, hc > 0 ? K / 4 : 0, f.st);
  if (hc == 0) return linear_tf32(dC, lin.t.t, out, M, K, N, nullptr, f.st);
  float* d = reinterpret_cast<float*>(f.ws.mg);
  int rc = linear_tf32(dC, lin.t.t, d, M, K, N, nullptr, f.st);
  return rc ? rc : launch_merge_scatter_add(d, out, f.images(), 2 * hc, 2 * wc, K / 4, f.st);
}

// The weight gradient of a token-stream Linear, dW [N, K] = dY^T X over M rows: exact fp32 (wgrad), or tf32 operands on the tensor cores.
// hc > 0: X is the fine stream of a TokenMerge over an hc x wc coarse grid, gathered 2x2 as the merge reads it (ldx unused).  The route
// is a flag, not a Fwd: kdb_wgrad calls this outside any forward.
int lin_dw(bool tf32, const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, int64_t M, int N, int K, float* part, cudaStream_t st,
           int hc = 0, int wc = 0) {
  if (hc > 0)
    return tf32 ? launch_wgrad_tf32_merge(dY, ldy, X, dW, M, N, hc, wc, K / 4, part, st)
                : launch_wgrad_merge(dY, ldy, X, dW, M, N, hc, wc, K / 4, part, st);
  return tf32 ? launch_wgrad_tf32(dY, ldy, X, ldx, dW, M, N, K, part, st) : launch_wgrad(dY, ldy, X, ldx, dW, M, N, K, part, st);
}

// The attention half's activations from the residual stream x, up to the attention output in ws.ao: the qkv projection goes to raw,
// the cosine-normalised and rotated q, k (with v) to ws.qkv.  The forward passes raw = ws.qkv and cosine-sim + RoPE runs in place (so
// on a JVP forward, where the tangent of q, k reads the projection, the raw tangent rows are in ws.qkv too); the reverse walk passes a
// buffer of its own, which keeps the projection for the cosine-sim VJP.  Routes in priority order (fp32 has only the last):
//   folded qkv GEMM: 1/rms from the row statistics, the AdaRMSNorm scale folded into the weight
//   RMSNorm + QKV_ROPE GEMM
//   RMSNorm + linear + qknorm_rope
template <typename T>
int attn_activations(KdbModel* m, Fwd& f, int k, const T* x, int h, int w, T* raw) {
  const LayerPlan& L = m->layers[k];
  const float* pos = f.pt->pos[L.level];
  const float2* rope = f.pt->rope[k];
  // M: primal token rows; Ma: every row of the token buffers (the tangent rows [M, 2M) follow on a JVP forward)
  const int64_t Ttok = (int64_t)h * w, M = (int64_t)f.B * Ttok, Ma = (int64_t)f.images() * Ttok;
  const int C = L.C;
  T* xn = reinterpret_cast<T*>(f.ws.xn);
  T* qkv = reinterpret_cast<T*>(f.ws.qkv);
  T* ao = reinterpret_cast<T*>(f.ws.ao);
  const std::string tag = "layer" + std::to_string(k);
  auto norm = [&] {
    int r = launch_rmsnorm<T>(x, xn, f.cond + L.ada_attn, f.cond_bs, Ttok, M, C, f.st);
    if constexpr (std::is_same_v<T, float>)
      if (!r && f.jvp) r = launch_rmsnorm_jvp(x, x + M * C, xn + M * C, f.cond + L.ada_attn, f.cond_bs, Ttok, M, C, f.st);
    return r ? r : m->tap<T>(tag + ".xn1", xn, Ma * C, f.st);
  };
  auto unfused = [&] {
    int r = norm();
    if (!r) r = lin_fwd<T>(f, xn, L.qkv, raw, Ma, GemmEpi{});
    // the tangent reads the un-normalised primal q and k, so it runs before the primal launch
    if constexpr (std::is_same_v<T, float>)
      if (!r && f.jvp) r = launch_qknorm_rope_jvp(raw, raw + M * 3 * C, pos, L.qr, M, (int)Ttok, L.nh, L.e, f.st);
    return r ? r : launch_qknorm_rope<T>(raw, qkv, pos, L.qr, M, (int)Ttok, L.nh, L.e, f.st);
  };
  int rc;
  if constexpr (std::is_same_v<T, bf16>) {
    GemmEpi qe;
    qe.mode = (L.e == 64 && rope != nullptr) ? EPI_QKV_ROPE : EPI_STORE;
    qe.C = C;
    qe.nh = L.nh;
    qe.T_tokens = (int)Ttok;
    qe.rope = rope;
    qe.qk_scale = L.qr.scale;
    qe.qk_eps = L.qr.eps;
    qe.rope_r = L.qr.R;
    GemmEpi qf = qe;
    qf.ss_in = f.ws.rowss;
    if (f.fold && f.stats && tc_gemm_supported(M, 3 * C, C, qf)) {
      rc = launch_gemm_tc(x, L.qkv_wf, qkv, M, 3 * C, C, qf, f.st);
      if (!rc && qf.mode == EPI_STORE) rc = launch_qknorm_rope<T>(qkv, qkv, pos, L.qr, M, (int)Ttok, L.nh, L.e, f.st);
    } else if (qe.mode == EPI_QKV_ROPE && tc_gemm_supported(M, 3 * C, C, qe)) {
      if (!(rc = norm())) rc = launch_gemm_tc(xn, L.qkv.wb, qkv, M, 3 * C, C, qe, f.st);
    } else {
      rc = unfused();
    }
  } else {
    rc = unfused();
  }
  if (rc || (rc = m->tap<T>(tag + ".qkv", qkv, Ma * 3 * C, f.st))) return rc;
  // q, k are normalised on every route above, so |q . k| <= scale: the attention kernels' fixed softmax shift when bounded
  if ((rc = attention_dispatch<T>(qkv, ao, f.B, h, w, L.nh, L.e, L.attn_type, L.attn_param, L.shift, f.st, L.bounded ? L.qr.scale : nullptr)))
    return rc;
  if constexpr (std::is_same_v<T, float>)
    if (f.jvp && (rc = launch_attention_jvp(qkv, qkv + M * 3 * C, ao + M * C, f.B, h, w, L.nh, L.e, L.attn_type, L.attn_param, L.shift, f.st)))
      return rc;
  return m->tap<T>(tag + ".ao", ao, Ma * C, f.st);
}

// The feed-forward half's up projection from the residual stream x: RMSNorm into ws.xn, up_proj into ws.hbuf.  The forward's unfused
// route and the reverse walk's recompute.
template <typename T>
int ff_up(KdbModel* m, Fwd& f, int k, const T* x, int h, int w) {
  const LayerPlan& L = m->layers[k];
  const int64_t Ttok = (int64_t)h * w, M = (int64_t)f.B * Ttok;
  const int C = L.C;
  T* xn = reinterpret_cast<T*>(f.ws.xn);
  int r = launch_rmsnorm<T>(x, xn, f.cond + L.ada_ff, f.cond_bs, Ttok, M, C, f.st);
  if constexpr (std::is_same_v<T, float>)
    if (!r && f.jvp) r = launch_rmsnorm_jvp(x, x + M * C, xn + M * C, f.cond + L.ada_ff, f.cond_bs, Ttok, M, C, f.st);
  return r ? r : lin_fwd<T>(f, xn, L.up, reinterpret_cast<T*>(f.ws.hbuf), f.images() * Ttok, GemmEpi{});
}

template <typename T>
int run_layer(KdbModel* m, Fwd& f, int k, T* x, int h, int w) {
  const LayerPlan& L = m->layers[k];
  const float2* rope = f.pt->rope[k];
  const int64_t Ttok = (int64_t)h * w, M = (int64_t)f.B * Ttok, Ma = (int64_t)f.images() * Ttok;
  const int C = L.C;
  T* hb = reinterpret_cast<T*>(f.ws.hbuf);
  T* gb = reinterpret_cast<T*>(f.ws.gbuf);
  const std::string tag = "layer" + std::to_string(k);
  int rc = 0;
  if (L.attn_type != KDB_ATTN_NONE) {
    if (f.tape) KDB_CUDA(cudaMemcpyAsync(f.tape[2 * k], x, sizeof(T) * M * C, cudaMemcpyDeviceToDevice, f.st));
    // attention: the whole half in one kernel (attn_block: 128-wide shifted-window levels; not while .qkv or .ao is tapped), or its
    // activations (attn_activations) and out_proj
    const bool block = f.fold && f.stats && rope != nullptr && !m->tapped(tag + ".qkv") && !m->tapped(tag + ".ao") &&
                       tc_attn_block_supported(h, w, C, L.nh, L.e, L.attn_type, L.attn_param, L.shift);
    if constexpr (std::is_same_v<T, bf16>) {
      if (block) {
        if ((rc = launch_attn_block(x, L.qkv_wf, L.out.wb, rope, L.qr.scale, f.B, h, w, L.shift, f.ws.rowss, f.ws.rowss, f.st))) return rc;
        f.stats = true;
      }
    }
    if (!block) {
      if ((rc = attn_activations<T>(m, f, k, x, h, w, reinterpret_cast<T*>(f.ws.qkv)))) return rc;
      GemmEpi e;
      e.mode = EPI_RESID;
      e.resid = x;
      f.produce(e, Ma, C, C);
      if ((rc = lin_fwd<T>(f, reinterpret_cast<T*>(f.ws.ao), L.out, x, Ma, e))) return rc;
    }
    if ((rc = m->tap<T>(tag + ".attn", x, Ma * C, f.st))) return rc;
  }
  if (f.tape) KDB_CUDA(cudaMemcpyAsync(f.tape[2 * k + 1], x, sizeof(T) * M * C, cudaMemcpyDeviceToDevice, f.st));
  auto unfused = [&] {
    int r = ff_up<T>(m, f, k, x, h, w);
    if (!r) r = launch_geglu<T>(hb, gb, M, L.dff, f.st);
    if constexpr (std::is_same_v<T, float>)
      if (!r && f.jvp) r = launch_geglu_jvp(hb, hb + M * 2 * L.dff, gb + M * L.dff, M, L.dff, f.st);
    return r;
  };
  // feed-forward, routes in priority order (fp32 has only the last):
  //   ffn_fused: the whole half in one kernel (128-wide levels; not while .geglu is tapped)
  //   folded GEGLU GEMM: 1/rms from the row statistics, the AdaRMSNorm scale folded into the weight
  //   RMSNorm + GEGLU GEMM
  //   RMSNorm + linear + geglu
  // then, after all but ffn_fused, down_proj
  const bool ffn = f.fold && f.stats && L.up_wf != nullptr && tc_ffn_fused_supported(M, C, L.dff) && !m->tapped(tag + ".geglu");
  if constexpr (std::is_same_v<T, bf16>) {
    T* xn = reinterpret_cast<T*>(f.ws.xn);
    GemmEpi ge;
    ge.mode = EPI_GEGLU;
    GemmEpi gf = ge;
    gf.ss_in = f.ws.rowss;
    if (ffn) {
      rc = launch_ffn_fused(x, L.up_wf, L.down.wb, M, C, L.dff, f.ws.rowss, f.ws.rowss, f.st);
      f.stats = true;
    } else if (f.fold && f.stats && L.up_wf != nullptr && tc_gemm_supported(M, 2 * L.dff, C, gf)) {
      rc = launch_gemm_tc(x, L.up_wf, gb, M, 2 * L.dff, C, gf, f.st);
    } else if (L.up_wb_il != nullptr && tc_gemm_supported(M, 2 * L.dff, C, ge)) {
      rc = launch_rmsnorm<T>(x, xn, f.cond + L.ada_ff, f.cond_bs, Ttok, M, C, f.st);
      if (!rc) rc = launch_gemm_tc(xn, L.up_wb_il, gb, M, 2 * L.dff, C, ge, f.st);
    } else {
      rc = unfused();
    }
  } else {
    rc = unfused();
  }
  if (rc) return rc;
  if (!ffn) {
    if ((rc = m->tap<T>(tag + ".geglu", gb, Ma * L.dff, f.st))) return rc;
    GemmEpi e;
    e.mode = EPI_RESID;
    e.resid = x;
    f.produce(e, Ma, C, L.dff);
    if ((rc = lin_fwd<T>(f, gb, L.down, x, Ma, e))) return rc;
  }
  return m->tap<T>(tag + ".ff", x, Ma * C, f.st);
}

// v != nullptr (fp32 only): forward-mode derivative along v, the tangent D'(x) v goes to out_t.  The primal launches are those of a
// plain forward of B images; the linear ones run over the tangent images as well (the SIMT GEMM's per-row arithmetic does not depend
// on M), each nonlinear one is followed by its tangent kernel.
// tape != nullptr (fp32 only): the residual stream entering every attention / feed-forward half and out_norm is copied to the tape
// (slots 2k, 2k+1 of layer k, slot 2 * layers for out_norm) for the reverse walk of kdb_model_forward_vjp; the launches are unchanged.
// pos_tables != nullptr: receives the position tables of this token grid.
// tf32 (fp32 only): the tf32 training route, every token-stream Linear through linear_tf32 on ensure_tf32's copies (lin_fwd).
template <typename T>
int forward_impl(KdbModel* m, int B, int H, int W, const float* x, const float* v, const float* sigma, float sd, const float* cond,
                 int64_t cond_bs, float* out, float* out_t, Workspace& ws, cudaStream_t st, float* const* tape = nullptr,
                 const PosTables** pos_tables = nullptr, bool tf32 = false) {
  constexpr bool kBf16 = std::is_same_v<T, bf16>;
  const KdbModelConfig& c = m->cfg;
  const int n = c.n_levels, C0 = c.width[0];
  const int h0 = H / c.patch_h, w0 = W / c.patch_w;
  PosTables* pt = nullptr;
  int rc = ensure_pos(m, h0, w0, st, &pt);
  if (rc || (tf32 && (rc = ensure_tf32(m, st)))) return rc;
  if (pos_tables) *pos_tables = pt;
  m->tap_count = 0;
  Fwd f{B, ws, st, cond, cond_bs, pt, kBf16 && m->fuse_norm, false, false, !kBf16 && v != nullptr};
  f.fold = f.emit && cond_bs == 0 && m->fold_descs != nullptr;
  f.tape = tape;
  f.tf32 = tf32;
  if (f.fold && (rc = launch_fold_norm_weights(m->fold_descs, m->n_fold, cond, st))) return rc;
  const int Bt = f.images();

  T* cur = reinterpret_cast<T*>(ws.xs[0]);
  auto patch_in = [&] {
    int r = launch_patch_in<T>(x, sigma, sd, m->patch_in_w, cur, B, c.in_channels, H, W, c.patch_h, c.patch_w, C0, st);
    // c_in x is linear in x: the tangent images are patch_in of v with the same sigma
    if (!r && f.jvp)
      r = launch_patch_in<T>(v, sigma, sd, m->patch_in_w, cur + (int64_t)B * h0 * w0 * C0, B, c.in_channels, H, W, c.patch_h, c.patch_w, C0, st);
    return r;
  };
  // patch_in: on the tensor core, which leaves the row statistics for the first fused RMSNorm, or the scalar kernel (other patch
  // geometries, where finalize made no patch_in_wb, and latents that start inside a 16-byte granule)
  if constexpr (kBf16) {
    if (m->patch_in_wb != nullptr && tc_patch_in_supported(x, C0, W)) {
      f.stats = f.emit;
      rc = launch_patch_in_tc(x, sigma, sd, m->patch_in_wb, cur, B, H, W, C0, f.stats ? ws.rowss : nullptr, st);
    } else {
      rc = patch_in();
    }
  } else {
    rc = patch_in();
  }
  if (rc || (rc = m->tap<T>("patch_in", cur, (int64_t)Bt * h0 * w0 * C0, st))) return rc;

  int k = 0, h = h0, w = w0;
  for (int l = 0; l < n - 1; ++l) {
    for (int i = 0; i < c.depth[l]; ++i)
      if ((rc = run_layer<T>(m, f, k++, cur, h, w))) return rc;
    if ((rc = m->tap<T>("L" + std::to_string(l) + ".down", cur, (int64_t)Bt * h * w * c.width[l], st))) return rc;
    T* nxt = reinterpret_cast<T*>(ws.xs[l + 1]);
    const int64_t Mc = (int64_t)Bt * (h / 2) * (w / 2);
    const int N = c.width[l + 1], K = 4 * c.width[l];
    auto merge = [&] {
      T* mg = reinterpret_cast<T*>(ws.mg);
      f.stats = false;
      int r = launch_merge_gather<T>(cur, mg, Bt, h, w, c.width[l], st);
      return r ? r : lin_fwd<T>(f, mg, m->merge[l], nxt, Mc, GemmEpi{});
    };
    // TokenMerge: the 2x2 gather rides on the GEMM's TMA loads when the geometry allows, else a gather kernel and a plain GEMM
    if constexpr (kBf16) {
      GemmEpi me;
      me.mC = c.width[l];
      me.mhc = h / 2;
      me.mwc = w / 2;
      if (tc_gemm_supported(Mc, N, K, me)) {
        f.produce(me, Mc, N, K);
        rc = launch_gemm_tc(cur, m->merge[l].wb, nxt, Mc, N, K, me, st);
      } else {
        rc = merge();
      }
    } else {
      rc = merge();
    }
    if (rc) return rc;
    h /= 2;
    w /= 2;
    if ((rc = m->tap<T>("L" + std::to_string(l) + ".merge", nxt, (int64_t)Bt * h * w * N, st))) return rc;
    cur = nxt;
  }
  for (int i = 0; i < c.depth[n - 1]; ++i)
    if ((rc = run_layer<T>(m, f, k++, cur, h, w))) return rc;
  if ((rc = m->tap<T>("mid", cur, (int64_t)Bt * h * w * c.width[n - 1], st))) return rc;
  for (int l = n - 2; l >= 0; --l) {
    T* up = reinterpret_cast<T*>(ws.xup[l]);
    GemmEpi e;
    e.mode = EPI_SPLIT_LERP;
    e.resid = ws.xs[l];
    e.fac = m->split_fac[l];
    e.hc = h;
    e.wc = w;
    e.C = c.width[l];
    f.produce(e, (int64_t)Bt * h * w, 4 * c.width[l], c.width[l + 1]);
    if ((rc = lin_fwd<T>(f, cur, m->split[l], up, (int64_t)Bt * h * w, e))) return rc;
    h *= 2;
    w *= 2;
    if ((rc = m->tap<T>("L" + std::to_string(l) + ".split", up, (int64_t)Bt * h * w * c.width[l], st))) return rc;
    for (int i = 0; i < c.depth[l]; ++i)
      if ((rc = run_layer<T>(m, f, k++, up, h, w))) return rc;
    if ((rc = m->tap<T>("L" + std::to_string(l) + ".up", up, (int64_t)Bt * h * w * c.width[l], st))) return rc;
    cur = up;
  }
  // patch_out, routes in priority order (fp32 has only the last):
  //   out_norm folded into the tensor-core projection, 1/rms from the row statistics
  //   out_norm as a row kernel, then the tensor-core projection
  //   the scalar kernel
  // The tensor-core epilogue un-patches and applies the Karras combine; it reads x and writes out as float4, so a view that starts
  // inside a 16-byte granule (a storage offset, a caller's out= buffer) takes the scalar kernel.
  if constexpr (kBf16) {
    const int64_t M0 = (int64_t)B * h0 * w0;
    GemmEpi pe;
    pe.mode = EPI_PATCH_OUT;
    pe.img = out;
    pe.x_in = x;
    pe.sigma = sigma;
    pe.sigma_data = sd;
    pe.H = H;
    pe.W = W;
    GemmEpi pf = pe;
    pf.ss_in = ws.rowss;
    if (f.stats && m->patch_out_wf != nullptr && tc_gemm_supported(M0, 64, C0, pf))
      return launch_gemm_tc(cur, m->patch_out_wf, nullptr, M0, 64, C0, pf, st);
    if (m->patch_out_wb != nullptr && tc_gemm_supported(M0, 64, C0, pe)) {
      bf16* xn = reinterpret_cast<bf16*>(ws.xn);
      if ((rc = launch_rmsnorm<bf16>(cur, xn, m->out_norm, 0, M0, M0, C0, st))) return rc;
      return launch_gemm_tc(xn, m->patch_out_wb, nullptr, M0, 64, C0, pe, st);
    }
  }
  if (tape)
    KDB_CUDA(cudaMemcpyAsync(tape[2 * m->layers.size()], cur, sizeof(T) * B * h0 * w0 * C0, cudaMemcpyDeviceToDevice, st));
  rc = launch_patch_out<T>(cur, m->out_norm, m->patch_out_w, x, sigma, sd, out, B, c.out_channels, H, W, c.patch_h, c.patch_w, C0, st);
  if constexpr (!kBf16)
    if (!rc && f.jvp)
      rc = launch_patch_out_jvp(cur, cur + (int64_t)B * h0 * w0 * C0, m->out_norm, m->patch_out_w, v, sigma, sd, out_t, B, c.out_channels, H, W,
                                c.patch_h, c.patch_w, C0, st);
  return rc;
}

// Reverse mode.  The workspace of kdb_model_forward_vjp is one fp32 forward workspace of B images followed by the tape (the residual
// stream entering every attention half, every feed-forward half and out_norm) and the gradient buffers.  The backward walk reuses the
// forward workspace's xn / qkv / ao / hbuf / mg buffers for the recomputed activations and as scratch.
struct VjpSpace {
  std::vector<float*> tape;   // 2 per layer (KdbModel::layers order; nullptr for the attention half of a layer without one) + out_norm
  std::vector<float*> g;      // per level: gradient of the residual stream [B, T_l, C_l]
  float *qkv_raw = nullptr;   // the qkv projection of the half being differentiated, before cosine-sim + RoPE
  float *dqkv = nullptr, *dbuf = nullptr, *dh = nullptr, *stats = nullptr;
  // kdb_model_forward_train only (carve_vjp with train): the AdaRMSNorm scale gradients [B, ada_total] (the layout of the conditioning
  // rows), the mapping network's output gradient [B, mw], its MapLayout rows, out_norm's rstd per token [B T0], the reduction partials
  float *dscale = nullptr, *dcond = nullptr, *map_keep = nullptr, *map_grad = nullptr, *rstd = nullptr, *part = nullptr;
  size_t total = 0;
};

void carve_vjp(const KdbModelConfig& c, int B, int H, int W, void* workspace, Workspace& ws, VjpSpace& vs, int ada_total = 0, bool train = false) {
  Carver cv(workspace, 1024);
  carve(c, KDB_PREC_FP32, B, H, W, cv, ws);
  cv.off = ws.total;
  auto take = [&](size_t floats) { return cv.take<float>(floats * sizeof(float)); };
  const int n = c.n_levels;
  const int64_t T0 = (int64_t)(H / c.patch_h) * (W / c.patch_w);
  auto stream_floats = [&](int l) { return (size_t)B * (T0 >> (2 * l)) * c.width[l]; };
  vs.tape.clear();
  for_each_layer(c, [&](const std::string&, int l, int) {
    vs.tape.push_back(c.attn_type[l] != KDB_ATTN_NONE ? take(stream_floats(l)) : nullptr);
    vs.tape.push_back(take(stream_floats(l)));
    return 0;
  });
  vs.tape.push_back(take(stream_floats(0)));
  vs.g.assign(n, nullptr);
  size_t mqkv = 0, md = 0, mh = 0, mst = 0;
  for (int l = 0; l < n; ++l) {
    vs.g[l] = take(stream_floats(l));
    const size_t toks = (size_t)B * (T0 >> (2 * l));
    md = std::max(md, toks * std::max(c.width[l], c.d_ff[l]));
    mh = std::max(mh, toks * 2 * c.d_ff[l]);
    if (c.attn_type[l] != KDB_ATTN_NONE) {
      mqkv = std::max(mqkv, 3 * stream_floats(l));
      mst = std::max(mst, toks * (c.width[l] / std::max(c.d_head[l], 1)) * 3);
    }
  }
  vs.qkv_raw = take(mqkv);
  vs.dqkv = take(mqkv);
  vs.dbuf = take(md);
  vs.dh = take(mh);
  vs.stats = take(mst);
  if (train) {
    const MapLayout ml{c.mapping_width, c.mapping_d_ff, c.mapping_depth};
    vs.dscale = take((size_t)B * ada_total);
    vs.dcond = take((size_t)B * c.mapping_width);
    vs.map_keep = take((size_t)B * ml.keep_floats());
    vs.map_grad = take((size_t)B * ml.grad_floats());
    vs.rstd = take((size_t)B * T0);
    vs.part = take((size_t)kTrainPartFloats);
  }
  vs.total = cv.total();
}

// What kdb_model_forward_train adds to the reverse walk besides the model's bound gradient buffers: its precision.
struct Train {
  bool tf32;   // KDB_PREC_TF32: the forward, the recomputes and every token-stream input and weight gradient take the tf32 route
};

// Layer k in reverse: g holds the gradient of the layer's output residual stream and receives that of its input.  Each half recomputes
// its activations from the tape with the forward's functions (ff_up, attn_activations; f is an fp32 forward of B images), runs the
// backward kernels and adds the branch gradient to g.
// tr != nullptr: also the gradients of the layer's weights, head scales and (into vs.dscale) AdaRMSNorm scales.
int vjp_layer(KdbModel* m, Fwd& f, VjpSpace& vs, int k, float* g, int h, int w, const Train* tr = nullptr) {
  const LayerPlan& L = m->layers[k];
  const int64_t Ttok = (int64_t)h * w, M = (int64_t)f.B * Ttok;
  const int C = L.C, F = L.dff;
  float* xn = reinterpret_cast<float*>(f.ws.xn);
  float* qkv = reinterpret_cast<float*>(f.ws.qkv);
  float* ao = reinterpret_cast<float*>(f.ws.ao);
  float* hb = reinterpret_cast<float*>(f.ws.hbuf);
  cudaStream_t st = f.st;
  int rc;
  // feed-forward half: x + down(geglu(up(norm(x))))
  const float* x = vs.tape[2 * k + 1];
  const std::string ff = L.prefix + "ff.", sa = L.prefix + "self_attn.";
  if ((rc = ff_up<float>(m, f, k, x, h, w))) return rc;
  if (tr) {   // down_proj's input, the GEGLU output
    float* gb = reinterpret_cast<float*>(f.ws.gbuf);
    if ((rc = launch_geglu<float>(hb, gb, M, F, st)) ||
        (rc = lin_dw(f.tf32, g, C, gb, F, m->grad(ff + "down_proj.weight"), M, C, F, vs.part, st)))
      return rc;
  }
  if ((rc = lin_dx(f, g, L.down, vs.dbuf, M))) return rc;
  if ((rc = launch_geglu_vjp(hb, vs.dbuf, vs.dh, M, F, st))) return rc;
  if (tr && (rc = lin_dw(f.tf32, vs.dh, 2 * F, xn, C, m->grad(ff + "up_proj.weight"), M, 2 * F, C, vs.part, st))) return rc;
  if ((rc = lin_dx(f, vs.dh, L.up, xn, M))) return rc;
  if (tr && (rc = launch_norm_scale_grad(x, C, xn, C, vs.dscale + L.ada_ff, m->ada_total, Ttok, M, C, vs.part, st))) return rc;
  if ((rc = launch_rmsnorm_vjp(x, xn, g, f.cond + L.ada_ff, f.cond_bs, Ttok, M, C, st))) return rc;
  if (L.attn_type == KDB_ATTN_NONE) return 0;
  // attention half: x + out(attn(qknorm_rope(qkv(norm(x)))))
  x = vs.tape[2 * k];
  if ((rc = attn_activations<float>(m, f, k, x, h, w, vs.qkv_raw))) return rc;
  if (tr && (rc = lin_dw(f.tf32, g, C, ao, C, m->grad(sa + "out_proj.weight"), M, C, C, vs.part, st))) return rc;
  if ((rc = lin_dx(f, g, L.out, vs.dbuf, M))) return rc;
  if ((rc = launch_attention_vjp(qkv, ao, vs.dbuf, vs.dqkv, vs.stats, f.B, h, w, L.nh, L.e, L.attn_type, L.attn_param, L.shift, st)))
    return rc;
  // the attention's statistics are spent: vs.stats takes the per-(row, head) terms of the head scales' gradient
  if ((rc = launch_qknorm_rope_vjp(vs.qkv_raw, vs.dqkv, f.pt->pos[L.level], L.qr, M, (int)Ttok, L.nh, L.e, st, tr ? vs.stats : nullptr)))
    return rc;
  if (tr && ((rc = launch_colsum(vs.stats, M, L.nh, m->grad(sa + "scale"), vs.part, st)) ||
             (rc = lin_dw(f.tf32, vs.dqkv, 3 * C, xn, C, m->grad(sa + "qkv_proj.weight"), M, 3 * C, C, vs.part, st))))
    return rc;
  if ((rc = lin_dx(f, vs.dqkv, L.qkv, xn, M))) return rc;
  if (tr && (rc = launch_norm_scale_grad(x, C, xn, C, vs.dscale + L.ada_attn, m->ada_total, Ttok, M, C, vs.part, st))) return rc;
  return launch_rmsnorm_vjp(x, xn, g, f.cond + L.ada_attn, f.cond_bs, Ttok, M, C, st);
}

// out = the fp32 forward (bit for bit: the same launches, plus the tape copies), then grad_x = u^T J(x) by a walk of the forward in
// reverse: patch_out + out_norm + combine; each up level's layers then its split-lerp; the mid layers; each down level (innermost
// first) its merge then its layers; patch_in.
// tr != nullptr (kdb_model_forward_train): along the walk, the gradients of patch_out, out_norm, every layer, split and merge, patch_in, and
// the AdaRMSNorm scales into vs.dscale; grad_x may then be nullptr.
int vjp_impl(KdbModel* m, int B, int H, int W, const float* x, const float* u, const float* sigma, float sd, const float* cond, int64_t cond_bs,
             float* out, float* grad_x, Workspace& ws, VjpSpace& vs, cudaStream_t st, const Train* tr = nullptr) {
  const PosTables* pt = nullptr;
  const bool tf32 = tr != nullptr && tr->tf32;
  int rc = forward_impl<float>(m, B, H, W, x, nullptr, sigma, sd, cond, cond_bs, out, nullptr, ws, st, vs.tape.data(), &pt, tf32);
  if (rc) return rc;
  const KdbModelConfig& c = m->cfg;
  const int n = c.n_levels, C0 = c.width[0];
  const int h0 = H / c.patch_h, w0 = W / c.patch_w;
  Fwd f{B, ws, st, cond, cond_bs, pt, false, false, false, false};
  f.tf32 = tf32;
  const int64_t M0 = (int64_t)B * h0 * w0;
  float* part = vs.part;
  // training: the backward also leaves out_norm's output gradient (ws.xn) and rstd; patch_out's weight gradient then reads its output
  // gradient (the patch rows of u) and its input (the out-normed stream) in place
  float* dnorm = tr ? reinterpret_cast<float*>(ws.xn) : nullptr;
  if ((rc = launch_patch_out_vjp(vs.tape.back(), m->out_norm, m->patch_out_w, u, sigma, sd, vs.g[0], B, c.out_channels, H, W, c.patch_h,
                                 c.patch_w, C0, st, dnorm, tr ? vs.rstd : nullptr)))
    return rc;
  if (tr && ((rc = launch_wgrad_patch_out(u, vs.tape.back(), m->out_norm, vs.rstd, m->grad("patch_out.proj.weight"), B, c.out_channels, H, W,
                                          c.patch_h, c.patch_w, C0, part, st)) ||
             (rc = launch_norm_scale_grad(vs.tape.back(), C0, dnorm, C0, m->grad("out_norm.scale"), 0, M0, M0, C0, part, st))))
    return rc;
  int k = (int)m->layers.size();
  float* mg = reinterpret_cast<float*>(ws.mg);
  for (int l = 0; l < n - 1; ++l) {
    const int h = h0 >> l, w = w0 >> l;
    for (int i = 0; i < c.depth[l]; ++i)
      if ((rc = vjp_layer(m, f, vs, --k, vs.g[l], h, w, tr))) return rc;
    // the split's input, the coarse stream it read: the mid level's output or the next level's up stream, both intact since the forward
    const float* coarse = reinterpret_cast<const float*>(l == n - 2 ? ws.xs[n - 1] : ws.xup[l + 1]);
    const int64_t Mc = (int64_t)B * (h / 2) * (w / 2);
    const std::string sp = "splits." + std::to_string(l) + ".";
    if (tr) {   // d fac = sum (y - skip) dup with y = the split projection recomputed (vs.dbuf), skip = ws.xs[l]
      if ((rc = lin_fwd<float>(f, coarse, m->split[l], vs.dbuf, Mc, GemmEpi{})) ||
          (rc = launch_split_fac_grad(vs.dbuf, reinterpret_cast<const float*>(ws.xs[l]), vs.g[l], m->grad(sp + "fac"), B, h, w, c.width[l],
                                      part, st)))
        return rc;
    }
    // up = lerp(skip, unpatch(cur W^T), fac): the coarse stream gets patch2x2(fac dup) W, the skip keeps (1 - fac) dup in g[l]
    if ((rc = launch_split_vjp_gather(vs.g[l], mg, m->split_fac[l], B, h, w, c.width[l], st))) return rc;
    if (tr && (rc = lin_dw(tf32, mg, 4 * c.width[l], coarse, c.width[l + 1], m->grad(sp + "proj.weight"), Mc, 4 * c.width[l], c.width[l + 1],
                           part, st)))
      return rc;
    if ((rc = lin_dx(f, mg, m->split[l], vs.g[l + 1], Mc))) return rc;
  }
  for (int i = 0; i < c.depth[n - 1]; ++i)
    if ((rc = vjp_layer(m, f, vs, --k, vs.g[n - 1], h0 >> (n - 1), w0 >> (n - 1), tr))) return rc;
  for (int l = n - 2; l >= 0; --l) {
    const int h = h0 >> l, w = w0 >> l;
    const int64_t Mc = (int64_t)B * (h / 2) * (w / 2);
    float* dmw = tr ? m->grad("merges." + std::to_string(l) + ".proj.weight") : nullptr;
    const float* fine = reinterpret_cast<const float*>(ws.xs[l]);
    if (dmw && (rc = lin_dw(tf32, vs.g[l + 1], c.width[l + 1], fine, c.width[l], dmw, Mc, c.width[l + 1], 4 * c.width[l], part, st, h / 2, w / 2)))
      return rc;
    // nxt = patch2x2(cur) W^T: the fine stream (already holding the skip gradient) gets unpatch2x2(dnxt W) added
    if ((rc = lin_dx(f, vs.g[l + 1], m->merge[l], vs.g[l], Mc, h / 2, w / 2))) return rc;
    for (int i = 0; i < c.depth[l]; ++i)
      if ((rc = vjp_layer(m, f, vs, --k, vs.g[l], h, w, tr))) return rc;
  }
  if (tr) {   // patch_in's input: the patch rows of x
    if ((rc = launch_wgrad_patch_in(vs.g[0], x, m->grad("patch_in.proj.weight"), B, c.in_channels, H, W, c.patch_h, c.patch_w, C0, part, st)))
      return rc;
    if (grad_x == nullptr) return 0;
  }
  return launch_patch_in_vjp(vs.g[0], m->patch_in_w, u, sigma, sd, grad_x, B, c.in_channels, H, W, c.patch_h, c.patch_w, C0, st);
}

// the class_cond / mapping_cond checks of kdb_model_conditioning, kdb_model_forward_train and kdb_model_mapping_vjp (image_transformer_v2.py:729-732)
int check_conds(const KdbModelConfig& c, const int64_t* class_cond, const float* mapping_cond) {
  KDB_REQUIRE(!(c.num_classes > 0 && class_cond == nullptr), KDB_ERR_BAD_ARG, "class_cond must be specified if num_classes > 0");
  KDB_REQUIRE(!(c.mapping_cond_dim > 0 && mapping_cond == nullptr), KDB_ERR_BAD_ARG, "mapping_cond must be specified if mapping_cond_dim > 0");
  return 0;
}

// the fine grid of the TokenSplit / TokenMerge elementwise entry points
int check_fine_grid(const char* what, int batch, int height, int width, int c) {
  KDB_REQUIRE(batch > 0 && c > 0, KDB_ERR_BAD_ARG, "%s: bad argument", what);
  KDB_REQUIRE(height >= 2 && width >= 2 && height % 2 == 0 && width % 2 == 0, KDB_ERR_BAD_SHAPE, "%s: %dx%d fine grid", what, height, width);
  return 0;
}

// an NCHW image of batch x channels x height x width in patch_h x patch_w patches, and Karras's sigma where sigma_data > 0
int check_patches(const char* what, int batch, int channels, int height, int width, int patch_h, int patch_w, float sigma_data,
                  const float* sigma) {
  KDB_REQUIRE(batch > 0 && channels > 0 && patch_h > 0 && patch_w > 0 && (sigma_data <= 0.f || sigma), KDB_ERR_BAD_ARG, "%s: bad argument", what);
  KDB_REQUIRE(height > 0 && width > 0 && height % patch_h == 0 && width % patch_w == 0, KDB_ERR_BAD_SHAPE, "%s: %dx%d image in %dx%d patches",
              what, height, width, patch_h, patch_w);
  return 0;
}

}  // namespace

extern "C" {

int kdb_model_create(const KdbModelConfig* cfg, KdbModel** out) {
  KDB_REQUIRE(cfg && out, KDB_ERR_BAD_ARG, "model_create: NULL argument");
  KDB_REQUIRE(cfg->n_levels >= 1 && cfg->n_levels <= KDB_MAX_LEVELS, KDB_ERR_BAD_ARG, "model_create: n_levels %d", cfg->n_levels);
  KDB_REQUIRE(cfg->patch_h >= 1 && cfg->patch_w >= 1 && cfg->in_channels >= 1 && cfg->out_channels >= 1, KDB_ERR_BAD_ARG,
              "model_create: bad patch/channels");
  KDB_REQUIRE(cfg->mapping_depth >= 0 && cfg->mapping_depth <= 8 && cfg->mapping_width >= 2, KDB_ERR_BAD_ARG, "model_create: bad mapping spec");
  KDB_REQUIRE(cfg->family == KDB_FAMILY_ITV2 || cfg->family == KDB_FAMILY_ITV1, KDB_ERR_BAD_ARG, "model_create: unknown model family %d", cfg->family);
  KDB_REQUIRE(cfg->family != KDB_FAMILY_ITV1 || (cfg->n_levels == 1 && cfg->attn_type[0] == KDB_ATTN_GLOBAL && cfg->d_head[0] == 64 &&
                                                 cfg->mapping_width == cfg->width[0] && cfg->mapping_cond_dim == 0),
              KDB_ERR_BAD_ARG, "model_create: image_transformer_v1 is one level of global attention, d_head 64, mapping width = width, no mapping_cond");
  for (int l = 0; l < cfg->n_levels; ++l) {
    KDB_REQUIRE(cfg->width[l] > 0 && cfg->depth[l] >= 0 && cfg->d_ff[l] > 0, KDB_ERR_BAD_ARG, "model_create: bad level %d", l);
    KDB_REQUIRE(cfg->attn_type[l] >= KDB_ATTN_NONE && cfg->attn_type[l] <= KDB_ATTN_SHIFTED_WINDOW, KDB_ERR_BAD_ARG,
                "model_create: unsupported self attention spec at level %d", l);
  }
  KdbModel* m = new KdbModel();
  m->cfg = *cfg;
  *out = m;
  return 0;
}

void kdb_model_destroy(KdbModel* m) { delete m; }

int kdb_model_set_tensor(KdbModel* m, const char* key, const float* data, const int64_t* shape, int ndim) {
  return set_tensor(m, key, data, shape, ndim);
}

int kdb_model_finalize(KdbModel* m, void* stream) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "finalize: NULL model");
  cudaStream_t st = (cudaStream_t)stream;
  m->free_all();
  m->pos_cache.clear();
  m->finalized = false;
  m->kept_ready = false;
  const KdbModelConfig& c = m->cfg;
  const int n = c.n_levels, mw = c.mapping_width;
  m->layers.clear();
  m->merge.assign(n, Lin{});
  m->split.assign(n, Lin{});
  m->split_fac.assign(n, nullptr);
  int ada = 0;
  int rc = for_each_layer(c, [&](const std::string& prefix, int level, int index) {
    m->layers.emplace_back();
    return plan_layer(m, m->layers.back(), prefix, level, index, &ada, st);
  });
  if (rc) return rc;
  m->ada_total = ada;
  {
    // table of (weights -> folded copy) pairs for the fused RMSNorm path
    std::vector<FoldDesc> descs;
    for (const LayerPlan& L : m->layers) {
      if (L.C % 8 != 0) continue;
      if (L.qkv_wf != nullptr && L.ada_attn >= 0) descs.push_back(FoldDesc{L.qkv.wb, L.qkv_wf, 3 * L.C, L.C, L.ada_attn});
      if (L.up_wf != nullptr && L.up_wb_il != nullptr) descs.push_back(FoldDesc{L.up_wb_il, L.up_wf, 2 * L.dff, L.C, L.ada_ff});
    }
    m->n_fold = (int)descs.size();
    m->fold_descs = nullptr;
    if (!descs.empty()) {
      if ((rc = m->alloc(&m->fold_descs, descs.size()))) return rc;
      KDB_CUDA(cudaMemcpyAsync(m->fold_descs, descs.data(), descs.size() * sizeof(FoldDesc), cudaMemcpyHostToDevice, st));
      KDB_CUDA(cudaStreamSynchronize(st));
    }
    const char* e = getenv("KDB200_NO_FUSED_NORM");
    m->fuse_norm = !(e != nullptr && e[0] == '1');
  }
  for (int l = 0; l < n - 1; ++l) {
    if ((rc = bind(m, m->merge[l], "merges." + std::to_string(l) + ".proj.weight", c.width[l + 1], 4 * c.width[l], st)) ||
        (rc = bind(m, m->split[l], "splits." + std::to_string(l) + ".proj.weight", 4 * c.width[l], c.width[l + 1], st)))
      return rc;
    GET("splits." + std::to_string(l) + ".fac", &m->split_fac[l], 1);
  }
  const int C0 = c.width[0], Np = c.patch_h * c.patch_w * c.out_channels, Ni = c.patch_h * c.patch_w * c.in_channels;
  GET("out_norm.scale", &m->out_norm, C0);
  if (c.family == KDB_FAMILY_ITV1) {   // in_proj / out_proj (image_transformer_v1.py:295,298) in the engine's patch feature order
    const float *wi, *wo;
    GET("in_proj.weight", &wi, C0, Ni);
    GET("out_proj.weight", &wo, Np, C0);
    std::vector<float> a, b((size_t)C0 * Ni);
    if ((rc = download(wi, (size_t)C0 * Ni, a, st))) return rc;
    for (int64_t r = 0; r < C0; ++r)
      for (int64_t n = 0; n < Ni; ++n) b[r * Ni + n] = a[r * Ni + v1_patch_feature(n, c.in_channels, c.patch_h, c.patch_w)];
    if ((rc = upload(m, b, &m->patch_in_w, st))) return rc;
    auto perm = [&](int64_t r) { return v1_patch_feature(r, c.out_channels, c.patch_h, c.patch_w); };
    if ((rc = permuted_rows(m, wo, Np, C0, perm, &m->patch_out_w, st))) return rc;
  } else {
    GET("patch_in.proj.weight", &m->patch_in_w, C0, Ni);
    GET("patch_out.proj.weight", &m->patch_out_w, Np, C0);
  }

  m->patch_in_wb = nullptr;
  if (c.in_channels == 3 && c.patch_h == 4 && c.patch_w == 4 && C0 % 128 == 0) {
    if ((rc = m->alloc(&m->patch_in_wb, (size_t)C0 * 64))) return rc;
    if ((rc = prepare_patch_in_weight(m->patch_in_w, m->patch_in_wb, C0, st))) return rc;
  }
  m->patch_out_wb = nullptr;
  m->patch_out_wf = nullptr;
  if (c.out_channels == 3 && c.patch_h == 4 && c.patch_w == 4) {   // zero-padded bf16 patch_out weight [64, C0] of the EPI_PATCH_OUT GEMM
    if ((rc = m->alloc(&m->patch_out_wb, (size_t)64 * C0))) return rc;
    KDB_CUDA(cudaMemsetAsync(m->patch_out_wb, 0, (size_t)64 * C0 * sizeof(bf16), st));
    if ((rc = launch_f32_to_bf16(m->patch_out_w, m->patch_out_wb, (int64_t)Np * C0, st))) return rc;
    if (C0 % 8 == 0) {   // out_norm.scale is a plain parameter: fold it once
      FoldDesc* d1 = nullptr;
      if ((rc = m->alloc(&m->patch_out_wf, (size_t)64 * C0))) return rc;
      if ((rc = m->alloc(&d1, 1))) return rc;
      const FoldDesc hd{m->patch_out_wb, m->patch_out_wf, 64, C0, 0};
      KDB_CUDA(cudaMemcpyAsync(d1, &hd, sizeof(FoldDesc), cudaMemcpyHostToDevice, st));
      if ((rc = launch_fold_norm_weights(d1, 1, m->out_norm, st))) return rc;
      KDB_CUDA(cudaStreamSynchronize(st));
    }
  }
  // conditioning weights
  CondWeights& w = m->cw;
  w = CondWeights{};
  w.mw = mw;
  w.depth = c.mapping_depth;
  w.dff = c.mapping_d_ff;
  w.n_classes = c.num_classes;
  w.mcond_dim = c.mapping_cond_dim;
  w.ada_total = ada;
  GET("time_emb.weight", &w.time_emb, mw / 2, 1);
  GET("time_in_proj.weight", &w.time_in, mw, mw);
  GET("aug_emb.weight", &w.aug_emb, mw / 2, 9);
  GET("aug_in_proj.weight", &w.aug_in, mw, mw);
  if (c.num_classes > 0) GET("class_emb.weight", &w.class_emb, c.num_classes, mw);
  if (c.mapping_cond_dim > 0) GET("mapping_cond_in_proj.weight", &w.mcond_in, mw, c.mapping_cond_dim);
  GET("mapping.in_norm.scale", &w.in_norm, mw);
  GET("mapping.out_norm.scale", &w.out_norm, mw);
  for (int i = 0; i < c.mapping_depth; ++i) {
    const std::string p = "mapping.blocks." + std::to_string(i) + ".";
    GET(p + "norm.scale", &w.blk_norm[i], mw);
    GET(p + "up_proj.weight", &w.blk_up[i], 2 * c.mapping_d_ff, mw);
    GET(p + "down_proj.weight", &w.blk_down[i], mw, c.mapping_d_ff);
  }
  // concatenated AdaRMSNorm projection [ada_total, mw]
  if ((rc = m->alloc(&m->ada_cat, (size_t)ada * mw))) return rc;
  for (const LayerPlan& L : m->layers) {
    if (L.ada_attn >= 0)
      KDB_CUDA(cudaMemcpyAsync(m->ada_cat + (size_t)L.ada_attn * mw, L.attn_norm_w, sizeof(float) * L.C * mw, cudaMemcpyDeviceToDevice, st));
    KDB_CUDA(cudaMemcpyAsync(m->ada_cat + (size_t)L.ada_ff * mw, L.ff_norm_w, sizeof(float) * L.C * mw, cudaMemcpyDeviceToDevice, st));
  }
  w.ada_cat = m->ada_cat;
  KDB_CUDA(cudaStreamSynchronize(st));
  m->finalized = true;
  return 0;
}

int64_t kdb_model_cond_stride(const KdbModel* m) {
  if (!m || !m->finalized) return KDB_ERR_NOT_FINAL;
  return (int64_t)align_up((size_t)(m->ada_total + m->cfg.mapping_width), 4);
}

int kdb_model_conditioning(KdbModel* m, int rows, const float* sigma, const float* aug_cond, const int64_t* class_cond,
                           const float* mapping_cond, float* cond_out, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "conditioning: model not finalized");
  KDB_REQUIRE(rows > 0 && sigma && cond_out, KDB_ERR_BAD_ARG, "conditioning: bad arguments");
  if (int rc = check_conds(m->cfg, class_cond, mapping_cond)) return rc;
  return launch_conditioning(m->cw, rows, sigma, aug_cond, class_cond, mapping_cond, cond_out, kdb_model_cond_stride(m),
                             (cudaStream_t)stream);
}

size_t kdb_model_workspace_bytes(const KdbModel* m, int precision, int batch, int height, int width) {
  if (!m || batch <= 0 || height <= 0 || width <= 0) return 0;
  if (precision == KDB_PREC_TF32 || precision == KDB_PREC_FP16) {
    set_error("model_workspace_bytes: the tf32 and fp16 precisions are built for the image_v1 U-Net only");
    return 0;
  }
  Workspace ws;
  Carver cv(nullptr, 1024);
  carve(m->cfg, precision, batch, height, width, cv, ws);
  return ws.total;
}

}  // extern "C"

namespace {

// image geometry and preconditioning checks shared by the forward entry points
int check_image(const KdbModel* m, const char* what, int height, int width, float sigma_data) {
  const KdbModelConfig& c = m->cfg;
  KDB_REQUIRE(height % c.patch_h == 0 && width % c.patch_w == 0, KDB_ERR_BAD_SHAPE, "%s: %dx%d not divisible by the patch size", what, height,
              width);
  const int div = 1 << (c.n_levels - 1);
  KDB_REQUIRE((height / c.patch_h) % div == 0 && (width / c.patch_w) % div == 0, KDB_ERR_BAD_SHAPE,
              "%s: token grid %dx%d not divisible by 2^(levels-1)", what, height / c.patch_h, width / c.patch_w);
  KDB_REQUIRE(!(sigma_data > 0.f && c.in_channels != c.out_channels), KDB_ERR_BAD_ARG, "%s: preconditioning needs C_in == C_out", what);
  return 0;
}

// carve a workspace of `images` token-stream images out of the caller's buffer
int carve_checked(const KdbModel* m, const char* what, int precision, int images, int height, int width, void* workspace, size_t workspace_bytes,
                  Workspace& ws) {
  Carver cv(workspace, 1024);
  carve(m->cfg, precision, images, height, width, cv, ws);
  KDB_REQUIRE(ws.total <= workspace_bytes, KDB_ERR_WORKSPACE, "%s: workspace %zu < required %zu", what, workspace_bytes, ws.total);
  return 0;
}

}  // namespace

extern "C" {

int kdb_model_forward(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* sigma,
                      float sigma_data, const float* cond, int64_t cond_batch_stride, float* out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "forward: model not finalized");
  KDB_REQUIRE(x && sigma && cond && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "forward: NULL argument");
  KDB_REQUIRE(precision != KDB_PREC_TF32 && precision != KDB_PREC_FP16, KDB_ERR_UNSUPPORTED,
              "forward: the tf32 and fp16 precisions are built for the image_v1 U-Net only");
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_BF16, KDB_ERR_BAD_ARG, "forward: bad precision %d", precision);
  int rc = check_image(m, "forward", height, width, sigma_data);
  if (rc) return rc;
  Workspace ws;
  if ((rc = carve_checked(m, "forward", precision, batch, height, width, workspace, workspace_bytes, ws))) return rc;
  if (precision == KDB_PREC_FP32)
    return m->disarm_tap(forward_impl<float>(m, batch, height, width, x, nullptr, sigma, sigma_data, cond, cond_batch_stride, out, nullptr,
                                             ws, (cudaStream_t)stream));
  return m->disarm_tap(forward_impl<bf16>(m, batch, height, width, x, nullptr, sigma, sigma_data, cond, cond_batch_stride, out, nullptr, ws,
                                          (cudaStream_t)stream));
}

int kdb_model_forward_jvp(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* v, const float* sigma,
                          float sigma_data, const float* cond, int64_t cond_batch_stride, float* out, float* out_tangent, void* workspace,
                          size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "forward_jvp: model not finalized");
  KDB_REQUIRE(x && v && sigma && cond && out && out_tangent && workspace && batch > 0, KDB_ERR_BAD_ARG, "forward_jvp: NULL argument");
  KDB_REQUIRE(precision == KDB_PREC_FP32, KDB_ERR_UNSUPPORTED, "forward_jvp: the derivative is built for the fp32 path only (precision %d)",
              precision);
  int rc = check_image(m, "forward_jvp", height, width, sigma_data);
  if (rc) return rc;
  Workspace ws;
  if ((rc = carve_checked(m, "forward_jvp", precision, 2 * batch, height, width, workspace, workspace_bytes, ws))) return rc;
  return m->disarm_tap(
      forward_impl<float>(m, batch, height, width, x, v, sigma, sigma_data, cond, cond_batch_stride, out, out_tangent, ws, (cudaStream_t)stream));
}

int64_t kdb_model_vjp_workspace_bytes(const KdbModel* m, int batch, int height, int width) {
  KDB_REQUIRE(m && batch > 0 && height > 0 && width > 0, KDB_ERR_BAD_ARG, "vjp_workspace_bytes: bad argument");
  Workspace ws;
  VjpSpace vs;
  carve_vjp(m->cfg, batch, height, width, nullptr, ws, vs);
  return (int64_t)vs.total;
}

int kdb_model_forward_vjp(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                          const float* cond, int64_t cond_batch_stride, const float* cotangent, float* out, float* grad_x, void* workspace,
                          size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "forward_vjp: model not finalized");
  KDB_REQUIRE(x && sigma && cond && cotangent && out && grad_x && workspace && batch > 0, KDB_ERR_BAD_ARG, "forward_vjp: NULL argument");
  KDB_REQUIRE(precision == KDB_PREC_FP32, KDB_ERR_UNSUPPORTED, "forward_vjp: the derivative is built for the fp32 path only (precision %d)",
              precision);
  int rc = check_image(m, "forward_vjp", height, width, sigma_data);
  if (rc) return rc;
  Workspace ws;
  VjpSpace vs;
  carve_vjp(m->cfg, batch, height, width, workspace, ws, vs);
  KDB_REQUIRE(vs.total <= workspace_bytes, KDB_ERR_WORKSPACE, "forward_vjp: workspace %zu < required %zu", workspace_bytes, vs.total);
  return m->disarm_tap(
      vjp_impl(m, batch, height, width, x, cotangent, sigma, sigma_data, cond, cond_batch_stride, out, grad_x, ws, vs, (cudaStream_t)stream));
}

}  // extern "C"

namespace {

// The transformer's refusal rule for a gradient buffer (check_grad): the tensors that are buffers, not parameters
int check_grad_key(const KdbModel*, const std::string& k) {
  const bool buffer = k == "time_emb.weight" || k == "aug_emb.weight" || (k.size() >= 13 && k.compare(k.size() - 13, 13, "pos_emb.freqs") == 0);
  KDB_REQUIRE(!buffer, KDB_ERR_BAD_ARG, "'%s' is a buffer, not a parameter", k.c_str());
  return 0;
}

// The precision of the training calls: KDB_PREC_FP32 or KDB_PREC_TF32, on image_transformer_v2 handles.  It needs no finalize, so the
// refusals come before the finalize check.
int check_training_precision(const KdbModel* m, const char* what, int precision) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "%s: NULL model", what);
  const KdbModelConfig& c = m->cfg;
  KDB_REQUIRE(c.family == KDB_FAMILY_ITV2, KDB_ERR_UNSUPPORTED,
              "%s: image_transformer_v1 runs on weights permuted and folded at finalize; its parameter gradients are not built", what);
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_TF32, KDB_ERR_UNSUPPORTED, "%s: training runs at fp32 or tf32 (precision %d)",
              what, precision);
  if (precision == KDB_PREC_TF32)
    for (int l = 0; l < c.n_levels; ++l)   // the tensor-core GEMM's TMA rows: 16-byte strides
      KDB_REQUIRE(c.width[l] % 4 == 0 && c.d_ff[l] % 4 == 0, KDB_ERR_UNSUPPORTED,
                  "%s: tf32 needs widths and d_ff that are multiples of 4 (level %d: %d, %d)", what, l, c.width[l], c.d_ff[l]);
  return 0;
}

}  // namespace

extern "C" {

int kdb_model_set_grad(KdbModel* m, const char* key, float* data, const int64_t* shape, int ndim) {
  return set_grad(m, "set_grad", key, data, shape, ndim, check_grad_key);
}

int64_t kdb_model_train_workspace_bytes(const KdbModel* m, int batch, int height, int width) {
  KDB_REQUIRE(m && batch > 0 && height > 0 && width > 0, KDB_ERR_BAD_ARG, "train_workspace_bytes: bad argument");
  KDB_REQUIRE(m->finalized, KDB_ERR_NOT_FINAL, "train_workspace_bytes: model not finalized");
  Workspace ws;
  VjpSpace vs;
  carve_vjp(m->cfg, batch, height, width, nullptr, ws, vs, m->ada_total, true);
  return (int64_t)vs.total;
}

int kdb_model_forward_train(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* sigma,
                            const float* aug_cond, const int64_t* class_cond, const float* mapping_cond, const float* cond,
                            int64_t cond_batch_stride, const float* cotangent, float* out, float* grad_x, void* workspace,
                            size_t workspace_bytes, void* stream) {
  int rc = check_training_precision(m, "forward_train", precision);
  if (rc) return rc;
  KDB_REQUIRE(m->finalized, KDB_ERR_NOT_FINAL, "forward_train: model not finalized");
  const KdbModelConfig& c = m->cfg;
  KDB_REQUIRE(x && sigma && cond && cotangent && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "forward_train: NULL argument");
  if ((rc = check_conds(c, class_cond, mapping_cond))) return rc;
  if ((rc = check_train(m, "forward_train", cond_batch_stride, kdb_model_cond_stride(m), check_grad_key))) return rc;
  if ((rc = check_image(m, "forward_train", height, width, 0.f))) return rc;
  Workspace ws;
  VjpSpace vs;
  carve_vjp(c, batch, height, width, workspace, ws, vs, m->ada_total, true);
  KDB_REQUIRE(vs.total <= workspace_bytes, KDB_ERR_WORKSPACE, "forward_train: workspace %zu < required %zu", workspace_bytes, vs.total);
  cudaStream_t st = (cudaStream_t)stream;
  const Train tr{precision == KDB_PREC_TF32};
  if ((rc = m->disarm_tap(vjp_impl(m, batch, height, width, x, cotangent, sigma, 0.f, cond, cond_batch_stride, out, grad_x, ws, vs, st, &tr))))
    return rc;
  // AdaRMSNorm: scale = 1 + cond W^T per image, so d W = sum_b dscale_b cond_b (cond: the last mw floats of the conditioning row) and the
  // mapping network's output gets dscale W over every layer at once (ada_cat: the layers' W stacked in the order of the scales)
  const int B = batch, mw = c.mapping_width, A = m->ada_total;
  const float* cond_vec = cond + A;
  float* part = vs.part;
  for (const LayerPlan& L : m->layers) {
    if (L.ada_attn >= 0 &&
        (rc = launch_wgrad(vs.dscale + L.ada_attn, A, cond_vec, cond_batch_stride, m->grad(L.prefix + "self_attn.norm.linear.weight"), B, L.C, mw,
                           part, st)))
      return rc;
    if ((rc = launch_wgrad(vs.dscale + L.ada_ff, A, cond_vec, cond_batch_stride, m->grad(L.prefix + "ff.norm.linear.weight"), B, L.C, mw, part, st)))
      return rc;
  }
  if ((rc = launch_gemm_vjp(vs.dscale, m->ada_cat, vs.dcond, B, A, mw, VJP_STORE, 0, 0, 0, st)) ||
      (rc = launch_mapping_backward(m->cw, B, sigma, aug_cond, class_cond, mapping_cond, vs.dcond, vs.map_keep, vs.map_grad, st)))
    return rc;
  // the mapping network's weights from the activations and gradients its backward left per row
  const MapLayout ml{mw, c.mapping_d_ff, c.mapping_depth};
  const int64_t K = ml.keep_floats(), G = ml.grad_floats();
  const float *keep = vs.map_keep, *grad = vs.map_grad;
  const int D = c.mapping_depth, F = c.mapping_d_ff;
  if ((rc = launch_norm_scale_grad(keep + ml.r(D), K, vs.dcond, mw, m->grad("mapping.out_norm.scale"), 0, B, B, mw, part, st))) return rc;
  for (int l = 0; l < D; ++l) {
    const std::string p = "mapping.blocks." + std::to_string(l) + ".";
    if ((rc = launch_norm_scale_grad(keep + ml.r(l), K, grad + ml.dxn(l), G, m->grad(p + "norm.scale"), 0, B, B, mw, part, st)) ||
        (rc = launch_wgrad(grad + ml.dh(l), G, keep + ml.xn(l), K, m->grad(p + "up_proj.weight"), B, 2 * F, mw, part, st)) ||
        (rc = launch_wgrad(grad + ml.dr(l + 1), G, keep + ml.g(l), K, m->grad(p + "down_proj.weight"), B, mw, F, part, st)))
      return rc;
  }
  const float* demb = grad + ml.demb();
  if ((rc = launch_norm_scale_grad(keep + ml.emb(), K, grad + ml.dr(0), G, m->grad("mapping.in_norm.scale"), 0, B, B, mw, part, st)) ||
      (rc = launch_wgrad(demb, G, keep + ml.ff_t(), K, m->grad("time_in_proj.weight"), B, mw, mw, part, st)) ||
      (rc = launch_wgrad(demb, G, keep + ml.ff_a(), K, m->grad("aug_in_proj.weight"), B, mw, mw, part, st)))
    return rc;
  if (c.mapping_cond_dim > 0 &&
      (rc = launch_wgrad(demb, G, mapping_cond, c.mapping_cond_dim, m->grad("mapping_cond_in_proj.weight"), B, mw, c.mapping_cond_dim, part, st)))
    return rc;
  if (c.num_classes > 0) return launch_class_emb_grad(demb, G, class_cond, m->grad("class_emb.weight"), B, c.num_classes, mw, st);
  return 0;
}

int kdb_model_train_forward(KdbModel* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                            const float* cond, int64_t cond_batch_stride, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_training_precision(m, "train_forward", precision);
  if (rc) return rc;
  KDB_REQUIRE(m->finalized, KDB_ERR_NOT_FINAL, "train_forward: model not finalized");
  KDB_REQUIRE(x && sigma && cond && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "train_forward: NULL argument");
  if ((rc = check_image(m, "train_forward", height, width, sigma_data))) return rc;
  Workspace ws;
  if ((rc = carve_checked(m, "train_forward", KDB_PREC_FP32, batch, height, width, workspace, workspace_bytes, ws))) return rc;
  return m->disarm_tap(forward_impl<float>(m, batch, height, width, x, nullptr, sigma, sigma_data, cond, cond_batch_stride, out, nullptr, ws,
                                           (cudaStream_t)stream, nullptr, nullptr, precision == KDB_PREC_TF32));
}

int kdb_wgrad(int precision, const float* dy, int64_t ldy, const float* x, int64_t ldx, float* dw, int64_t m, int n, int k, int merge_hc,
              int merge_wc, float* scratch, void* stream) {
  KDB_REQUIRE(dy && x && dw && scratch && m > 0 && n > 0 && k > 0, KDB_ERR_BAD_ARG, "wgrad: bad argument");
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_TF32, KDB_ERR_UNSUPPORTED, "wgrad: precision %d is neither fp32 nor tf32",
              precision);
  KDB_REQUIRE(ldy >= n, KDB_ERR_BAD_ARG, "wgrad: ldy %lld < n %d", (long long)ldy, n);
  if (merge_hc > 0 || merge_wc > 0)
    KDB_REQUIRE(merge_hc > 0 && merge_wc > 0 && k % 4 == 0 && m % ((int64_t)merge_hc * merge_wc) == 0, KDB_ERR_BAD_SHAPE,
                "wgrad: merge geometry %dx%d with k %d, m %lld", merge_hc, merge_wc, k, (long long)m);
  else
    KDB_REQUIRE(ldx >= k, KDB_ERR_BAD_ARG, "wgrad: ldx %lld < k %d", (long long)ldx, k);
  return lin_dw(precision == KDB_PREC_TF32, dy, ldy, x, ldx, dw, m, n, k, scratch, (cudaStream_t)stream, merge_hc, merge_wc);
}

int kdb_wgrad_patch_in(const float* dtok, const float* x, float* dw, int batch, int channels, int height, int width, int patch_h, int patch_w,
                       int n, float* scratch, void* stream) {
  KDB_REQUIRE(dtok && x && dw && scratch && batch > 0 && channels > 0 && n > 0 && patch_h > 0 && patch_w > 0, KDB_ERR_BAD_ARG,
              "wgrad_patch_in: bad argument");
  KDB_REQUIRE(height > 0 && width > 0 && height % patch_h == 0 && width % patch_w == 0, KDB_ERR_BAD_SHAPE,
              "wgrad_patch_in: %dx%d image in %dx%d patches", height, width, patch_h, patch_w);
  return launch_wgrad_patch_in(dtok, x, dw, batch, channels, height, width, patch_h, patch_w, n, scratch, (cudaStream_t)stream);
}

int kdb_wgrad_patch_out(const float* u, const float* tokens, const float* scale, const float* rstd, float* dw, int batch, int channels,
                        int height, int width, int patch_h, int patch_w, int c0, float* scratch, void* stream) {
  KDB_REQUIRE(u && tokens && scale && rstd && dw && scratch && batch > 0 && channels > 0 && c0 > 0 && patch_h > 0 && patch_w > 0,
              KDB_ERR_BAD_ARG, "wgrad_patch_out: bad argument");
  KDB_REQUIRE(height > 0 && width > 0 && height % patch_h == 0 && width % patch_w == 0, KDB_ERR_BAD_SHAPE,
              "wgrad_patch_out: %dx%d image in %dx%d patches", height, width, patch_h, patch_w);
  return launch_wgrad_patch_out(u, tokens, scale, rstd, dw, batch, channels, height, width, patch_h, patch_w, c0, scratch, (cudaStream_t)stream);
}

int kdb_norm_scale_grad(const float* x, int64_t ldx, const float* dy, int64_t ldy, float* out, int64_t ldo, int64_t rows_per_image,
                        int64_t rows, int c, float* scratch, void* stream) {
  KDB_REQUIRE(x && dy && out && scratch && c > 0 && ldx >= c && ldy >= c, KDB_ERR_BAD_ARG, "norm_scale_grad: bad argument");
  KDB_REQUIRE(rows_per_image == rows || ldo >= c, KDB_ERR_BAD_ARG, "norm_scale_grad: ldo %lld < c %d with several images", (long long)ldo, c);
  return launch_norm_scale_grad(x, ldx, dy, ldy, out, ldo, rows_per_image, rows, c, scratch, (cudaStream_t)stream);
}

int kdb_colsum(const float* p, int64_t rows, int c, float* out, float* scratch, void* stream) {
  KDB_REQUIRE(p && out && scratch && rows > 0 && c > 0, KDB_ERR_BAD_ARG, "colsum: bad argument");
  return launch_colsum(p, rows, c, out, scratch, (cudaStream_t)stream);
}

int kdb_variance_loss(const float* x, const float* noise, const float* sigma, float sigma_data, const float* f, const float* logvar, float* loss,
                      float* cotangent, float* dlogvar, int batch, int64_t per_sample, void* stream) {
  return launch_variance_loss(x, noise, sigma, sigma_data, f, logvar, loss, cotangent, dlogvar, batch, per_sample, (cudaStream_t)stream);
}

int kdb_split_fac_grad(const float* y, const float* skip, const float* dup, float* out, int batch, int height, int width, int c, float* scratch,
                       void* stream) {
  KDB_REQUIRE(y && skip && dup && out && scratch && batch > 0 && c > 0, KDB_ERR_BAD_ARG, "split_fac_grad: bad argument");
  KDB_REQUIRE(height >= 2 && width >= 2 && height % 2 == 0 && width % 2 == 0, KDB_ERR_BAD_SHAPE, "split_fac_grad: %dx%d fine grid", height,
              width);
  return launch_split_fac_grad(y, skip, dup, out, batch, height, width, c, scratch, (cudaStream_t)stream);
}

int kdb_class_emb_grad(const float* demb, int64_t ldd, const int64_t* cls, float* out, int rows, int n_classes, int mw, void* stream) {
  KDB_REQUIRE(demb && cls && out && rows > 0 && n_classes > 0 && mw > 0 && ldd >= mw, KDB_ERR_BAD_ARG, "class_emb_grad: bad argument");
  return launch_class_emb_grad(demb, ldd, cls, out, rows, n_classes, mw, (cudaStream_t)stream);
}

int kdb_gemm_vjp(const float* dc, const float* w, float* out, int64_t m, int n, int k, int epi, int hc, int wc, int cf, void* stream) {
  KDB_REQUIRE(dc && w && out && m > 0 && n > 0 && k > 0, KDB_ERR_BAD_ARG, "gemm_vjp: bad argument");
  KDB_REQUIRE(epi == VJP_STORE || epi == VJP_UNPATCH_ACC, KDB_ERR_BAD_ARG, "gemm_vjp: bad epilogue %d", epi);
  KDB_REQUIRE(epi == VJP_STORE || (hc > 0 && wc > 0 && cf > 0), KDB_ERR_BAD_ARG, "gemm_vjp: un-patch grid %dx%d of %d channels", hc, wc, cf);
  return launch_gemm_vjp(dc, w, out, m, n, k, epi, hc, wc, cf, (cudaStream_t)stream);
}

int kdb_rmsnorm_vjp(const float* x, const float* dy, float* dx, const float* scale, int64_t scale_bstride, int64_t rows_per_image, int64_t rows,
                    int c, void* stream) {
  KDB_REQUIRE(x && dy && dx && scale && rows > 0 && c > 0 && rows_per_image > 0 && scale_bstride >= 0, KDB_ERR_BAD_ARG,
              "rmsnorm_vjp: bad argument");
  KDB_REQUIRE(ceil_div(rows, 8) <= INT32_MAX, KDB_ERR_BAD_SHAPE, "rmsnorm_vjp: %lld rows", (long long)rows);
  return launch_rmsnorm_vjp(x, dy, dx, scale, scale_bstride, rows_per_image, rows, c, (cudaStream_t)stream);
}

int kdb_qknorm_rope_vjp(const float* qkv, float* dqkv, const float* pos, const float* freqs, const float* scale, float eps, int r, int64_t rows,
                        int t_tokens, int n_heads, int d_head, float* dscale_rows, void* stream) {
  KDB_REQUIRE(qkv && dqkv && pos && freqs && scale && rows > 0 && t_tokens > 0 && n_heads > 0 && eps >= 0.f, KDB_ERR_BAD_ARG,
              "qknorm_rope_vjp: bad argument");
  KDB_REQUIRE(rows % t_tokens == 0 && ceil_div(rows * n_heads, 4) <= INT32_MAX, KDB_ERR_BAD_SHAPE, "qknorm_rope_vjp: %lld rows of %d tokens",
              (long long)rows, t_tokens);
  QkRope qr;
  qr.freqs = freqs, qr.scale = scale, qr.eps = eps, qr.R = r;
  return launch_qknorm_rope_vjp(qkv, dqkv, pos, qr, rows, t_tokens, n_heads, d_head, (cudaStream_t)stream, dscale_rows);
}

int kdb_geglu_vjp(const float* h, const float* dy, float* dh, int64_t m, int f, void* stream) {
  KDB_REQUIRE(h && dy && dh && m > 0 && f > 0, KDB_ERR_BAD_ARG, "geglu_vjp: bad argument");
  return launch_geglu_vjp(h, dy, dh, m, f, (cudaStream_t)stream);
}

int kdb_split_vjp_gather(float* dup, float* out, const float* fac, int batch, int height, int width, int c, void* stream) {
  KDB_REQUIRE(dup && out && fac, KDB_ERR_BAD_ARG, "split_vjp_gather: NULL argument");
  if (int rc = check_fine_grid("split_vjp_gather", batch, height, width, c)) return rc;
  return launch_split_vjp_gather(dup, out, fac, batch, height, width, c, (cudaStream_t)stream);
}

int kdb_split_unpatch_lerp(const float* y, const float* skip, const float* fac, float* up, int batch, int height, int width, int c, void* stream) {
  KDB_REQUIRE(y && skip && fac && up, KDB_ERR_BAD_ARG, "split_unpatch_lerp: NULL argument");
  if (int rc = check_fine_grid("split_unpatch_lerp", batch, height, width, c)) return rc;
  return launch_split_unpatch_lerp(y, skip, fac, up, batch, height, width, c, (cudaStream_t)stream);
}

int kdb_merge_scatter_add(const float* d, float* dfine, int batch, int height, int width, int c, void* stream) {
  KDB_REQUIRE(d && dfine, KDB_ERR_BAD_ARG, "merge_scatter_add: NULL argument");
  if (int rc = check_fine_grid("merge_scatter_add", batch, height, width, c)) return rc;
  return launch_merge_scatter_add(d, dfine, batch, height, width, c, (cudaStream_t)stream);
}

int kdb_patch_out_vjp(const float* tokens, const float* norm_scale, const float* w, const float* u, const float* sigma, float sigma_data,
                      float* dtokens, int batch, int channels, int height, int width, int patch_h, int patch_w, int c0, float* dnorm, float* rstd,
                      void* stream) {
  KDB_REQUIRE(tokens && norm_scale && w && u && dtokens && c0 > 0, KDB_ERR_BAD_ARG, "patch_out_vjp: bad argument");
  if (int rc = check_patches("patch_out_vjp", batch, channels, height, width, patch_h, patch_w, sigma_data, sigma)) return rc;
  return launch_patch_out_vjp(tokens, norm_scale, w, u, sigma, sigma_data, dtokens, batch, channels, height, width, patch_h, patch_w, c0,
                              (cudaStream_t)stream, dnorm, rstd);
}

int kdb_patch_in_vjp(const float* dtokens, const float* w, const float* u, const float* sigma, float sigma_data, float* grad_x, int batch,
                     int channels, int height, int width, int patch_h, int patch_w, int n, void* stream) {
  KDB_REQUIRE(dtokens && w && grad_x && n > 0 && (sigma_data <= 0.f || u), KDB_ERR_BAD_ARG, "patch_in_vjp: bad argument");
  if (int rc = check_patches("patch_in_vjp", batch, channels, height, width, patch_h, patch_w, sigma_data, sigma)) return rc;
  return launch_patch_in_vjp(dtokens, w, u, sigma, sigma_data, grad_x, batch, channels, height, width, patch_h, patch_w, n, (cudaStream_t)stream);
}

int kdb_model_mapping_vjp(const KdbModel* m, int rows, const float* sigma, const float* aug_cond, const int64_t* class_cond,
                          const float* mapping_cond, const float* dcond, float* keep, float* grad, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "model_mapping_vjp: model NULL or not finalized");
  KDB_REQUIRE(rows > 0 && sigma && dcond && keep && grad, KDB_ERR_BAD_ARG, "model_mapping_vjp: bad argument");
  if (int rc = check_conds(m->cfg, class_cond, mapping_cond)) return rc;
  return launch_mapping_backward(m->cw, rows, sigma, aug_cond, class_cond, mapping_cond, dcond, keep, grad, (cudaStream_t)stream);
}

int kdb_model_debug_tap(KdbModel* m, const char* name, float* out, int64_t capacity) { return arm_tap(m, name, out, capacity); }

int64_t kdb_model_tap_count(const KdbModel* m) { return m ? m->tap_count : 0; }

int kdb_attention(int precision, int fast, const void* qkv, void* out, int batch, int h, int w, int n_heads, int d_head, int attn_type,
                  int attn_param, int shift, const float* logit_bound, void* stream) {
  KDB_REQUIRE(qkv && out && batch > 0 && h > 0 && w > 0 && n_heads > 0 && d_head > 0, KDB_ERR_BAD_ARG, "attention: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == KDB_PREC_TF32) {   // the image_v1 U-Net's global attention on fp32 tensors (q pre-scaled), d_head 64
    KDB_REQUIRE(attn_type == KDB_ATTN_GLOBAL && !fast, KDB_ERR_UNSUPPORTED, "attention: tf32 is built for global attention only");
    return launch_unet_attn_tf32(static_cast<const float*>(qkv), static_cast<float*>(out), batch, h * w, n_heads, d_head, st);
  }
  if (precision == KDB_PREC_FP16) {   // the same at fp16
    KDB_REQUIRE(attn_type == KDB_ATTN_GLOBAL && !fast, KDB_ERR_UNSUPPORTED, "attention: fp16 is built for global attention only");
    return launch_unet_attn_fp16(static_cast<const float*>(qkv), static_cast<float*>(out), batch, h * w, n_heads, d_head, st);
  }
  if (precision == KDB_PREC_FP32) {
    KDB_REQUIRE(!fast, KDB_ERR_UNSUPPORTED, "attention: tensor-core path is bf16 only");
    return launch_attention_generic<float>(static_cast<const float*>(qkv), static_cast<float*>(out), batch, h, w, n_heads, d_head,
                                           attn_type, attn_param, shift, st);
  }
  if (fast) {
    KDB_REQUIRE(tc_attention_supported(h, w, n_heads, d_head, attn_type, attn_param), KDB_ERR_UNSUPPORTED,
                "attention: shape not covered by the tensor-core kernels");
    return launch_attention_tc(static_cast<const bf16*>(qkv), static_cast<bf16*>(out), batch, h, w, n_heads, d_head, attn_type,
                               attn_param, shift, st, logit_bound);
  }
  return launch_attention_generic<bf16>(static_cast<const bf16*>(qkv), static_cast<bf16*>(out), batch, h, w, n_heads, d_head, attn_type,
                                        attn_param, shift, st);
}

int kdb_attention_jvp(const float* qkv, const float* dqkv, float* dout, int batch, int h, int w, int n_heads, int d_head, int attn_type,
                      int attn_param, int shift, void* stream) {
  KDB_REQUIRE(qkv && dqkv && dout && batch > 0 && h > 0 && w > 0 && n_heads > 0 && d_head > 0, KDB_ERR_BAD_ARG,
              "attention_jvp: bad argument");
  return launch_attention_jvp(qkv, dqkv, dout, batch, h, w, n_heads, d_head, attn_type, attn_param, shift, (cudaStream_t)stream);
}

int kdb_attention_vjp(const float* qkv, const float* out, const float* dout, float* dqkv, float* stats, int batch, int h, int w, int n_heads,
                      int d_head, int attn_type, int attn_param, int shift, void* stream) {
  KDB_REQUIRE(qkv && out && dout && dqkv && stats && batch > 0 && h > 0 && w > 0 && n_heads > 0 && d_head > 0, KDB_ERR_BAD_ARG,
              "attention_vjp: bad argument");
  return launch_attention_vjp(qkv, out, dout, dqkv, stats, batch, h, w, n_heads, d_head, attn_type, attn_param, shift, (cudaStream_t)stream);
}

}  // extern "C"
