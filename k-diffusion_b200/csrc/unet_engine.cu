// unet_engine.cu -- host-side execution plan of the image_v1 U-Net denoiser, on the exact fp32 path or with its convolutions and
// attention at tf32 or fp16
// (reference: k_diffusion/models/image_v1.py, layers.py:116-313, augmentation.py:92-104).
//
// Like the transformer engine, it owns no activations: the caller passes one workspace and the forward carves it.  Weights are
// borrowed device pointers keyed by the state-dict names of ImageDenoiserModelV1; kdb_unet_finalize builds the derived tables
// (tap-major convolution weights and their tf32- and fp16-rounded copies, the attention scale folded into qkv_proj's q rows, the concatenated
// AdaGN mappers).
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "model_core.cuh"
#include "unet_kernels.cuh"

namespace {

enum ModKind { M_RES = 0, M_ATTN, M_DOWN, M_UP, M_CONCAT };

// the derived (owned) copies of one conv weight: tap-major fp32, and that rounded to tf32 and to fp16
struct ConvW {
  const float* f32 = nullptr;
  const float* tf32 = nullptr;
  const __half* f16 = nullptr;
};

// One module of the U-Net in execution order.  M_CONCAT starts a UBlock that receives the matching skip.
struct UMod {
  int kind = M_RES, level = 0;
  std::string tap;
  int c_in = 0, c_mid = 0, c_out = 0;
  int groups1 = 1, groups2 = 1, ada1 = 0, ada2 = 0;
  ConvW w1, w2, skip_w;
  const float *b1 = nullptr, *b2 = nullptr;   // derived (owned) biases
  const float *mapper1_w = nullptr, *mapper1_b = nullptr, *mapper2_w = nullptr, *mapper2_b = nullptr;
  bool to_skip = false;           // the last module of a DBlock writes the level's skip buffer
};

}  // namespace

struct KdbUNet : kdb::ModelCore {
  KdbUNetConfig cfg{};
  std::vector<UMod> mods;
  const float *proj_in_w = nullptr, *proj_in_b = nullptr, *proj_out_w = nullptr, *proj_out_b = nullptr;
  int ada_total = 0;
  kdb::UNetCondWeights cw{};
};

using namespace kdb;

namespace {

// owned tap-major copy of a conv weight [N, C, ks, ks], the first scaled_rows output rows times scale, and that copy rounded to tf32
// and to fp16
int conv_weight(KdbUNet* m, const std::string& key, int N, int C, int ks, ConvW* out, cudaStream_t st, int scaled_rows = 0,
                float scale = 1.f) {
  const float* src;
  GET(key, &src, N, C, ks, ks);
  const size_t n = (size_t)N * C * ks * ks;
  float *dst = nullptr, *dst_tf32 = nullptr;
  __half* dst_f16 = nullptr;
  int rc = m->alloc(&dst, n);
  if (rc || (rc = m->alloc(&dst_tf32, n)) || (rc = m->alloc(&dst_f16, (size_t)N * ks * ks * f16_weight_ld(C))) ||
      (rc = launch_unet_reorder_conv_weight(src, dst, N, C, ks, scaled_rows, scale, st)) ||
      (rc = launch_unet_round_tf32(dst, dst_tf32, (int64_t)n, st)) || (rc = launch_unet_round_f16(dst, dst_f16, (int64_t)N * ks * ks, C, st)))
    return rc;
  *out = ConvW{dst, dst_tf32, dst_f16};
  return 0;
}

int bias_copy(KdbUNet* m, const std::string& key, int N, const float** out, cudaStream_t st, int scaled_rows = 0, float scale = 1.f) {
  const float* src;
  GET(key, &src, N);
  float* dst = nullptr;
  int rc = m->alloc(&dst, (size_t)N);
  if (rc || (rc = launch_unet_reorder_conv_weight(src, dst, N, 1, 1, scaled_rows, scale, st))) return rc;
  *out = dst;
  return 0;
}

// AdaGN mapper of `prefix` (Linear feats_in -> 2C with bias): bound and given the next offset of the conditioning row
int mapper(KdbUNet* m, const std::string& prefix, int C, const float** w, const float** b, int* off) {
  const int mw = m->cfg.mapping_out;
  GET(prefix + "mapper.weight", w, 2 * C, mw);
  GET(prefix + "mapper.bias", b, 2 * C);
  *off = m->ada_total;
  m->ada_total += 2 * C;
  return 0;
}

int plan_res(KdbUNet* m, const std::string& p, UMod& u, cudaStream_t st) {
  int rc;
  if ((rc = mapper(m, p + "main.0.", u.c_in, &u.mapper1_w, &u.mapper1_b, &u.ada1))) return rc;
  if ((rc = conv_weight(m, p + "main.2.weight", u.c_mid, u.c_in, 3, &u.w1, st))) return rc;
  if ((rc = bias_copy(m, p + "main.2.bias", u.c_mid, &u.b1, st))) return rc;
  if ((rc = mapper(m, p + "main.4.", u.c_mid, &u.mapper2_w, &u.mapper2_b, &u.ada2))) return rc;
  if ((rc = conv_weight(m, p + "main.6.weight", u.c_out, u.c_mid, 3, &u.w2, st))) return rc;
  if ((rc = bias_copy(m, p + "main.6.bias", u.c_out, &u.b2, st))) return rc;
  if (u.c_in != u.c_out && (rc = conv_weight(m, p + "skip.weight", u.c_out, u.c_in, 1, &u.skip_w, st))) return rc;
  u.groups1 = std::max(1, u.c_in / 32);
  u.groups2 = std::max(1, u.c_mid / 32);
  return 0;
}

// SelfAttention2d: softmax's 1/sqrt(d_head) is folded into the q rows of qkv_proj (weight and bias)
int plan_attn(KdbUNet* m, const std::string& p, UMod& u, cudaStream_t st) {
  int rc;
  const int C = u.c_out, nh = std::max(1, C / 64);
  const float scale = 1.f / std::sqrt((float)(C / nh));
  if ((rc = mapper(m, p + "norm_in.", C, &u.mapper1_w, &u.mapper1_b, &u.ada1))) return rc;
  if ((rc = conv_weight(m, p + "qkv_proj.weight", 3 * C, C, 1, &u.w1, st, C, scale))) return rc;
  if ((rc = bias_copy(m, p + "qkv_proj.bias", 3 * C, &u.b1, st, C, scale))) return rc;
  if ((rc = conv_weight(m, p + "out_proj.weight", C, C, 1, &u.w2, st))) return rc;
  if ((rc = bias_copy(m, p + "out_proj.bias", C, &u.b2, st))) return rc;
  u.groups1 = std::max(1, C / 32);
  return 0;
}

// DBlock / UBlock modules (image_v1.py:33-68): ResConvBlock [+ SelfAttention2d] per layer
int plan_block(KdbUNet* m, const std::string& p, int level, const char* tag, int depth, int c_in, int c_mid, int c_out, bool attn, int first,
               cudaStream_t st) {
  int idx = first, rc;
  for (int i = 0; i < depth; ++i) {
    UMod r;
    r.kind = M_RES;
    r.level = level;
    r.c_in = i == 0 ? c_in : c_mid;
    r.c_mid = c_mid;
    r.c_out = i < depth - 1 ? c_mid : c_out;
    r.tap = std::string(tag) + std::to_string(level) + "." + std::to_string(idx);
    if ((rc = plan_res(m, p + std::to_string(idx) + ".", r, st))) return rc;
    m->mods.push_back(r);
    ++idx;
    if (attn) {
      UMod a;
      a.kind = M_ATTN;
      a.level = level;
      a.c_in = a.c_mid = a.c_out = r.c_out;
      a.tap = std::string(tag) + std::to_string(level) + "." + std::to_string(idx);
      if ((rc = plan_attn(m, p + std::to_string(idx) + ".", a, st))) return rc;
      m->mods.push_back(a);
      ++idx;
    }
  }
  return 0;
}

// Workspace: the skip buffer of every level, then seven working buffers of `elems` floats each (two for the block stream, the
// AdaGN output, the first conv's output, the skip conv's output, qkv and the attention output).
struct UWs {
  float* skip[KDB_MAX_LEVELS] = {};
  float *x[2] = {}, *n1 = nullptr, *n2 = nullptr, *s = nullptr, *qkv = nullptr, *ao = nullptr;
  size_t total = 0;
};

void level_dims(const KdbUNetConfig& c, int H, int W, int l, int* h, int* w) {
  *h = H / c.patch_size;
  *w = W / c.patch_size;
  for (int i = c.skip_stages; i < l; ++i) {
    *h /= 2;
    *w /= 2;
  }
}

void carve(const KdbUNetConfig& c, int B, int H, int W, void* workspace, UWs& ws) {
  Carver cv(workspace, 256);
  auto take = [&](size_t floats) { return cv.take<float>(floats * sizeof(float)); };
  size_t elems = 0;
  for (int l = c.skip_stages; l < c.n_levels; ++l) {
    int h, w;
    level_dims(c, H, W, l, &h, &w);
    const size_t px = (size_t)B * h * w;
    ws.skip[l] = take(px * c.channels[l]);
    const size_t wide = std::max({3 * c.channels[l], 2 * c.channels[l], c.channels[std::max(0, l - 1)]});
    elems = std::max(elems, px * wide);
  }
  ws.x[0] = take(elems);
  ws.x[1] = take(elems);
  ws.n1 = take(elems);
  ws.n2 = take(elems);
  ws.s = take(elems);
  ws.qkv = take(elems);
  ws.ao = take(elems);
  ws.total = cv.total();
}

// the block input: one tensor, or a tensor and the matching skip (the UBlock concat)
struct Src {
  const float* p1 = nullptr;
  int c1 = 0;
  const float* p2 = nullptr;
  int c2 = 0;
};

// a convolution at the forward's precision, on the copy of its weight made for that precision
int conv(int prec, ConvArgs a, const ConvW& w, int ks, cudaStream_t st) {
  if (prec == KDB_PREC_FP16) return launch_unet_conv_fp16(a, w.f16, ks, st);
  if (prec == KDB_PREC_TF32) {
    a.w = w.tf32;
    return launch_unet_conv_tf32(a, ks, st);
  }
  a.w = w.f32;
  return launch_unet_conv(a, ks, st);
}

int run_res(int prec, const UMod& u, const Src& in, float* out, UWs& ws, int B, int h, int w, const float* cond, int64_t cbs, cudaStream_t st) {
  int rc;
  if ((rc = launch_unet_adagn(in.p1, in.c1, in.p2, in.c2, ws.n1, cond, cbs, u.ada1, u.groups1, true, B, h * w, st))) return rc;
  ConvArgs a;
  a.B = B, a.H = h, a.W = w;
  a.in1 = ws.n1, a.c1 = u.c_in, a.bias = u.b1, a.out = ws.n2, a.N = u.c_mid;
  if ((rc = conv(prec, a, u.w1, 3, st))) return rc;
  if ((rc = launch_unet_adagn(ws.n2, u.c_mid, nullptr, 0, ws.n1, cond, cbs, u.ada2, u.groups2, true, B, h * w, st))) return rc;
  ConvArgs c2;
  c2.B = B, c2.H = h, c2.W = w;
  if (u.skip_w.f32 != nullptr) {
    ConvArgs s;
    s.B = B, s.H = h, s.W = w;
    s.in1 = in.p1, s.c1 = in.c1, s.in2 = in.p2, s.c2 = in.c2, s.out = ws.s, s.N = u.c_out;
    if ((rc = conv(prec, s, u.skip_w, 1, st))) return rc;
    c2.r1 = ws.s, c2.rc1 = u.c_out;
  } else {
    c2.r1 = in.p1, c2.rc1 = in.c1, c2.r2 = in.p2;
  }
  c2.in1 = ws.n1, c2.c1 = u.c_mid, c2.bias = u.b2, c2.out = out, c2.N = u.c_out;
  return conv(prec, c2, u.w2, 3, st);
}

int run_attn(int prec, const UMod& u, const float* x, float* out, UWs& ws, int B, int h, int w, const float* cond, int64_t cbs, cudaStream_t st) {
  int rc;
  const int C = u.c_out, nh = std::max(1, C / 64);
  if ((rc = launch_unet_adagn(x, C, nullptr, 0, ws.n1, cond, cbs, u.ada1, u.groups1, false, B, h * w, st))) return rc;
  ConvArgs q;
  q.B = B, q.H = h, q.W = w;
  q.in1 = ws.n1, q.c1 = C, q.bias = u.b1, q.out = ws.qkv, q.N = 3 * C;
  if ((rc = conv(prec, q, u.w1, 1, st))) return rc;
  // at tf32 and fp16 the tensor-core attention takes the head size it is built for (64, that of every reference config); others keep
  // attn_generic
  if (prec == KDB_PREC_TF32 && unet_attn_tc_supported(C / nh))
    rc = launch_unet_attn_tf32(ws.qkv, ws.ao, B, h * w, nh, C / nh, st);
  else if (prec == KDB_PREC_FP16 && unet_attn_tc_supported(C / nh))
    rc = launch_unet_attn_fp16(ws.qkv, ws.ao, B, h * w, nh, C / nh, st);
  else
    rc = launch_attention_generic<float>(ws.qkv, ws.ao, B, h, w, nh, C / nh, KDB_ATTN_GLOBAL, 0, 0, st);
  if (rc) return rc;
  ConvArgs o;
  o.B = B, o.H = h, o.W = w;
  o.in1 = ws.ao, o.c1 = C, o.bias = u.b2, o.r1 = x, o.rc1 = C, o.out = out, o.N = C;
  return conv(prec, o, u.w2, 1, st);
}

int unet_forward(KdbUNet* m, int prec, int B, int H, int W, const float* x, const float* sigma, float sd, const float* cond, int64_t cbs, float* out,
                 UWs& ws, cudaStream_t st) {
  const KdbUNetConfig& c = m->cfg;
  const int s0 = c.skip_stages, C0 = c.channels[std::max(0, s0 - 1)];
  int h, w, rc;
  level_dims(c, H, W, s0, &h, &w);
  if ((rc = launch_unet_patch_in(x, sigma, sd, m->proj_in_w, m->proj_in_b, ws.x[0], B, c.in_channels, H, W, c.patch_size, C0, st))) return rc;
  if ((rc = m->tap("patch_in", ws.x[0], (int64_t)B * h * w * C0, st))) return rc;
  Src cur{ws.x[0], C0, nullptr, 0};
  int cur_buf = 0;                         // index of the ping-pong buffer holding cur (-1: a skip buffer)
  for (const UMod& u : m->mods) {
    const int nb = cur_buf == 0 ? 1 : 0;
    float* dst = u.to_skip ? ws.skip[u.level] : ws.x[nb];
    int C = u.c_out;
    switch (u.kind) {
      case M_DOWN:
        if ((rc = launch_unet_resample(cur.p1, dst, B, h, w, cur.c1, false, st))) return rc;
        h /= 2, w /= 2, C = cur.c1;
        break;
      case M_UP:
        if ((rc = launch_unet_resample(cur.p1, dst, B, h, w, cur.c1, true, st))) return rc;
        h *= 2, w *= 2, C = cur.c1;
        break;
      case M_CONCAT:
        cur.p2 = ws.skip[u.level], cur.c2 = c.channels[u.level];
        continue;
      case M_RES:
        if ((rc = run_res(prec, u, cur, dst, ws, B, h, w, cond, cbs, st))) return rc;
        break;
      default:
        if ((rc = run_attn(prec, u, cur.p1, dst, ws, B, h, w, cond, cbs, st))) return rc;
    }
    if ((rc = m->tap(u.tap, dst, (int64_t)B * h * w * C, st))) return rc;
    cur = Src{dst, C, nullptr, 0};
    cur_buf = u.to_skip ? -1 : nb;
  }
  return launch_unet_patch_out(cur.p1, m->proj_out_w, m->proj_out_b, x, sigma, sd, out, B, c.in_channels, H, W, c.patch_size, cur.c1, st);
}

}  // namespace

extern "C" {

int kdb_unet_create(const KdbUNetConfig* cfg, KdbUNet** out) {
  KDB_REQUIRE(cfg && out, KDB_ERR_BAD_ARG, "unet_create: NULL argument");
  KDB_REQUIRE(cfg->n_levels >= 1 && cfg->n_levels <= KDB_MAX_LEVELS, KDB_ERR_BAD_ARG, "unet_create: n_levels %d", cfg->n_levels);
  KDB_REQUIRE(cfg->in_channels >= 1 && cfg->patch_size >= 1 && cfg->mapping_out >= 2 && cfg->mapping_out % 2 == 0, KDB_ERR_BAD_ARG,
              "unet_create: bad channels / patch size / mapping_out");
  KDB_REQUIRE(cfg->skip_stages >= 0 && cfg->skip_stages < cfg->n_levels, KDB_ERR_BAD_ARG, "unet_create: skip_stages %d", cfg->skip_stages);
  KDB_REQUIRE(cfg->mapping_cond_dim >= (cfg->augment_wrapper ? 9 : 0), KDB_ERR_BAD_ARG,
              "unet_create: the augment wrapper needs mapping_cond_dim >= 9");
  for (int l = 0; l < cfg->n_levels; ++l) {
    KDB_REQUIRE(cfg->depth[l] >= 1 && cfg->channels[l] >= 4 && cfg->channels[l] % 4 == 0, KDB_ERR_UNSUPPORTED,
                "unet_create: level %d needs depth >= 1 and a channel count that is a multiple of 4", l);
    // a self-attention level attends at channels[l] and, in its UBlock's last layer, at channels[l - 1] (layers.py:184 asserts both)
    for (int C : {cfg->channels[l], cfg->channels[std::max(0, l - 1)]})
      KDB_REQUIRE(!cfg->self_attn[l] || C % std::max(1, C / 64) == 0, KDB_ERR_BAD_ARG,
                  "unet_create: level %d self-attention width %d is not divisible by its %d heads", l, C, std::max(1, C / 64));
  }
  KdbUNet* m = new KdbUNet();
  m->cfg = *cfg;
  *out = m;
  return 0;
}

int kdb_unet_destroy(KdbUNet* m) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "unet_destroy: NULL handle");
  delete m;
  return 0;
}

int kdb_unet_set_tensor(KdbUNet* m, const char* key, const float* data, const int64_t* shape, int ndim) {
  return set_tensor(m, key, data, shape, ndim);
}

int kdb_unet_finalize(KdbUNet* m, void* stream) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "unet_finalize: NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  m->free_all();
  m->finalized = false;
  m->mods.clear();
  m->ada_total = 0;
  const KdbUNetConfig& c = m->cfg;
  const int n = c.n_levels, s0 = c.skip_stages, mw = c.mapping_out, C0 = c.channels[std::max(0, s0 - 1)];
  int rc;
  for (int l = s0; l < n; ++l) {          // DBlocks (image_v1.py:108-110); module 0 downsamples when l > skip_stages
    if (l > s0) {
      UMod d;
      d.kind = M_DOWN, d.level = l, d.tap = "d" + std::to_string(l) + ".down";
      m->mods.push_back(d);
    }
    if ((rc = plan_block(m, "u_net.d_blocks." + std::to_string(l) + ".", l, "d", c.depth[l], c.channels[std::max(0, l - 1)], c.channels[l],
                         c.channels[l], c.self_attn[l] != 0, 1, st)))
      return rc;
    m->mods.back().to_skip = true;
  }
  for (int l = n - 1; l >= s0; --l) {     // UBlocks innermost first (layers.py:310-311); u_net.u_blocks.k holds level n-1-k
    if (l < n - 1) {
      UMod cc;
      cc.kind = M_CONCAT, cc.level = l;
      m->mods.push_back(cc);
    }
    const int c_in = l < n - 1 ? 2 * c.channels[l] : c.channels[l];
    if ((rc = plan_block(m, "u_net.u_blocks." + std::to_string(n - 1 - l) + ".", l, "u", c.depth[l], c_in, c.channels[l],
                         c.channels[std::max(0, l - 1)], c.self_attn[l] != 0, 0, st)))
      return rc;
    if (l > s0) {
      UMod up;
      up.kind = M_UP, up.level = l, up.tap = "u" + std::to_string(l) + ".up";
      m->mods.push_back(up);
    }
  }
  const int Kin = c.in_channels * c.patch_size * c.patch_size, Kout = Kin + (c.has_variance ? 1 : 0);
  GET("proj_in.weight", &m->proj_in_w, C0, Kin, 1, 1);
  GET("proj_in.bias", &m->proj_in_b, C0);
  GET("proj_out.weight", &m->proj_out_w, Kout, C0, 1, 1);
  GET("proj_out.bias", &m->proj_out_b, Kout);
  // conditioning weights and the concatenated AdaGN mappers
  UNetCondWeights& w = m->cw;
  w = UNetCondWeights{};
  w.mw = mw, w.mcond_dim = c.mapping_cond_dim, w.augment = c.augment_wrapper, w.ada_total = m->ada_total;
  GET("timestep_embed.weight", &w.time_emb, mw / 2, 1);
  if (c.mapping_cond_dim > 0) GET("mapping_cond.weight", &w.mcond_w, mw, c.mapping_cond_dim);
  GET("mapping.0.weight", &w.map_w0, mw, mw);
  GET("mapping.0.bias", &w.map_b0, mw);
  GET("mapping.2.weight", &w.map_w1, mw, mw);
  GET("mapping.2.bias", &w.map_b1, mw);
  float *aw, *ab;
  if ((rc = m->alloc(&aw, (size_t)m->ada_total * mw)) || (rc = m->alloc(&ab, (size_t)m->ada_total))) return rc;
  for (const UMod& u : m->mods) {
    const int n_ada = u.kind == M_RES ? 2 : (u.kind == M_ATTN ? 1 : 0);
    for (int i = 0; i < n_ada; ++i) {
      const int off = i ? u.ada2 : u.ada1, C = i ? u.c_mid : (u.kind == M_RES ? u.c_in : u.c_out);
      KDB_CUDA(cudaMemcpyAsync(aw + (size_t)off * mw, i ? u.mapper2_w : u.mapper1_w, sizeof(float) * 2 * C * mw, cudaMemcpyDeviceToDevice, st));
      KDB_CUDA(cudaMemcpyAsync(ab + off, i ? u.mapper2_b : u.mapper1_b, sizeof(float) * 2 * C, cudaMemcpyDeviceToDevice, st));
    }
  }
  w.ada_w = aw, w.ada_b = ab;
  KDB_CUDA(cudaStreamSynchronize(st));
  m->finalized = true;
  return 0;
}

int64_t kdb_unet_cond_stride(const KdbUNet* m) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "unet_cond_stride: model NULL or not finalized");
  return (int64_t)align_up((size_t)(m->ada_total + m->cfg.mapping_out), 4);
}

int kdb_unet_conditioning(KdbUNet* m, int rows, const float* sigma, const float* aug_cond, const float* mapping_cond, float* cond_out,
                          void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "unet_conditioning: model NULL or not finalized");
  KDB_REQUIRE(rows > 0 && sigma && cond_out, KDB_ERR_BAD_ARG, "unet_conditioning: bad arguments");
  const KdbUNetConfig& c = m->cfg;
  KDB_REQUIRE(!(aug_cond && !c.augment_wrapper), KDB_ERR_BAD_ARG, "unet_conditioning: aug_cond needs the augment wrapper");
  KDB_REQUIRE(!(c.augment_wrapper && c.mapping_cond_dim > 9 && mapping_cond == nullptr), KDB_ERR_BAD_ARG,
              "unet_conditioning: mapping_cond must be given (mapping_cond_dim %d)", c.mapping_cond_dim - 9);
  KDB_REQUIRE(!(mapping_cond && c.mapping_cond_dim == (c.augment_wrapper ? 9 : 0)), KDB_ERR_BAD_ARG,
              "unet_conditioning: the model takes no mapping_cond");
  return launch_unet_conditioning(m->cw, rows, sigma, aug_cond, mapping_cond, cond_out, kdb_unet_cond_stride(m), (cudaStream_t)stream);
}

int64_t kdb_unet_workspace_bytes(const KdbUNet* m, int precision, int batch, int height, int width) {
  KDB_REQUIRE(m && batch > 0 && height > 0 && width > 0, KDB_ERR_BAD_ARG, "unet_workspace_bytes: bad argument");
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_TF32 || precision == KDB_PREC_FP16, KDB_ERR_UNSUPPORTED,
              "unet_workspace_bytes: the fp32, tf32 and fp16 paths are built (precision %d)", precision);
  UWs ws;
  carve(m->cfg, batch, height, width, nullptr, ws);
  return (int64_t)ws.total;
}

int kdb_unet_forward(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                     const float* cond, int64_t cond_batch_stride, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "unet_forward: model NULL or not finalized");
  KDB_REQUIRE(x && sigma && cond && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "unet_forward: NULL argument");
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_TF32 || precision == KDB_PREC_FP16, KDB_ERR_UNSUPPORTED,
              "unet_forward: the fp32, tf32 and fp16 paths are built (precision %d)", precision);
  const KdbUNetConfig& c = m->cfg;
  KDB_REQUIRE(height > 0 && width > 0 && height % c.patch_size == 0 && width % c.patch_size == 0, KDB_ERR_BAD_SHAPE,
              "unet_forward: %dx%d not divisible by the patch size %d", height, width, c.patch_size);
  for (int l = c.skip_stages; l < c.n_levels; ++l) {
    int h, w;
    level_dims(c, height, width, l, &h, &w);
    const bool down_from = l < c.n_levels - 1;        // this grid is downsampled, and the upsample must restore it
    KDB_REQUIRE(h >= 2 && w >= 2 && (!down_from || (h % 2 == 0 && w % 2 == 0)), KDB_ERR_BAD_SHAPE,
                "unet_forward: level %d grid %dx%d (every level but the innermost needs an even grid, every level >= 2x2)", l, h, w);
  }
  UWs ws;
  carve(c, batch, height, width, workspace, ws);
  KDB_REQUIRE(ws.total <= workspace_bytes, KDB_ERR_WORKSPACE, "unet_forward: workspace %zu < required %zu", workspace_bytes, ws.total);
  return m->disarm_tap(unet_forward(m, precision, batch, height, width, x, sigma, sigma_data, cond, cond_batch_stride, out, ws, (cudaStream_t)stream));
}

int kdb_unet_debug_tap(KdbUNet* m, const char* name, float* out, int64_t capacity) { return arm_tap(m, name, out, capacity); }

int64_t kdb_unet_tap_count(const KdbUNet* m) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "unet_tap_count: NULL handle");
  return m->tap_count;
}

int kdb_unet_conv(const float* in1, int c1, const float* in2, int c2, const float* w_tapmajor, const float* bias, const float* r1, int rc1,
                  const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream) {
  ConvArgs a;
  a.in1 = in1, a.c1 = c1, a.in2 = in2, a.c2 = c2, a.w = w_tapmajor, a.bias = bias, a.r1 = r1, a.rc1 = rc1, a.r2 = r2, a.out = out;
  a.B = batch, a.H = h, a.W = w, a.N = n_out;
  return launch_unet_conv(a, ksize, (cudaStream_t)stream);
}

int kdb_unet_conv_tf32(const float* in1, int c1, const float* in2, int c2, const float* w_tapmajor, const float* bias, const float* r1,
                       int rc1, const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream) {
  ConvArgs a;
  a.in1 = in1, a.c1 = c1, a.in2 = in2, a.c2 = c2, a.w = w_tapmajor, a.bias = bias, a.r1 = r1, a.rc1 = rc1, a.r2 = r2, a.out = out;
  a.B = batch, a.H = h, a.W = w, a.N = n_out;
  return launch_unet_conv_tf32(a, ksize, (cudaStream_t)stream);
}

int kdb_unet_conv_fp16(const float* in1, int c1, const float* in2, int c2, const void* w_tapmajor_f16, const float* bias, const float* r1,
                       int rc1, const float* r2, float* out, int batch, int h, int w, int n_out, int ksize, void* stream) {
  ConvArgs a;
  a.in1 = in1, a.c1 = c1, a.in2 = in2, a.c2 = c2, a.bias = bias, a.r1 = r1, a.rc1 = rc1, a.r2 = r2, a.out = out;
  a.B = batch, a.H = h, a.W = w, a.N = n_out;
  return launch_unet_conv_fp16(a, static_cast<const __half*>(w_tapmajor_f16), ksize, (cudaStream_t)stream);
}

}  // extern "C"
