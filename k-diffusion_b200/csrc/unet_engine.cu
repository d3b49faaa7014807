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
  std::string prefix;             // state-dict prefix of a ResConvBlock or SelfAttention2d
  ConvW w1, w2, skip_w;
  const float *w1t = nullptr, *w2t = nullptr, *skip_t = nullptr;   // the input-gradient weights (ensure_bwd)
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
    r.prefix = p + std::to_string(idx) + ".";
    if ((rc = plan_res(m, p + std::to_string(idx) + ".", r, st))) return rc;
    m->mods.push_back(r);
    ++idx;
    if (attn) {
      UMod a;
      a.kind = M_ATTN;
      a.level = level;
      a.c_in = a.c_mid = a.c_out = r.c_out;
      a.tap = std::string(tag) + std::to_string(level) + "." + std::to_string(idx);
      a.prefix = p + std::to_string(idx) + ".";
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

// The one walk over the modules in execution order: fn(i, module, input, grid h, w before it, h, w after it, output channels, out) runs or
// sizes module i and sets out to the buffer it wrote (x0: patch_in's output).  walk makes that the next module's input, and a DBlock's
// last module's output the skip its level's UBlock concatenates.  M_CONCAT takes no call.
template <typename Fn>
int walk(const KdbUNet* m, int H, int W, float* x0, Fn fn) {
  const KdbUNetConfig& c = m->cfg;
  int h, w;
  level_dims(c, H, W, c.skip_stages, &h, &w);
  Src cur{x0, c.channels[std::max(0, c.skip_stages - 1)], nullptr, 0};
  float* skip[KDB_MAX_LEVELS] = {};
  for (size_t i = 0; i < m->mods.size(); ++i) {
    const UMod& u = m->mods[i];
    if (u.kind == M_CONCAT) {
      cur.p2 = skip[u.level], cur.c2 = c.channels[u.level];
      continue;
    }
    const int h0 = h, w0 = w;
    int C = u.c_out;
    if (u.kind == M_DOWN) h /= 2, w /= 2, C = cur.c1;
    if (u.kind == M_UP) h *= 2, w *= 2, C = cur.c1;
    float* dst = nullptr;
    if (int rc = fn(i, u, cur, h0, w0, h, w, C, dst)) return rc;
    if (u.to_skip) skip[u.level] = dst;
    cur = Src{dst, C, nullptr, 0};
  }
  return 0;
}

// tape != nullptr (training): patch_in writes tape[0] and module i (of m->mods) tape[i + 1], which a DBlock's last module's UBlock then reads
// as its skip; the launches are those of tape == nullptr.  logvar != nullptr (a has_variance model): the variance row's token mean per image
// after patch_out, from the same features.
int unet_forward(KdbUNet* m, int prec, int B, int H, int W, const float* x, const float* sigma, float sd, const float* cond, int64_t cbs, float* out,
                 UWs& ws, cudaStream_t st, float* const* tape = nullptr, float* logvar = nullptr) {
  const KdbUNetConfig& c = m->cfg;
  const int s0 = c.skip_stages, C0 = c.channels[std::max(0, s0 - 1)];
  int h, w, rc;
  level_dims(c, H, W, s0, &h, &w);
  float* y = tape ? tape[0] : ws.x[0];   // patch_in's output, then each module's in turn
  if ((rc = launch_unet_patch_in(x, sigma, sd, m->proj_in_w, m->proj_in_b, y, B, c.in_channels, H, W, c.patch_size, C0, st))) return rc;
  if ((rc = m->tap("patch_in", y, (int64_t)B * h * w * C0, st))) return rc;
  // without a tape, a module writes its level's skip buffer or the ping-pong buffer its input is not in
  rc = walk(m, H, W, y, [&](size_t i, const UMod& u, const Src& in, int hi, int wi, int ho, int wo, int C, float*& dst) {
    dst = tape ? tape[i + 1] : u.to_skip ? ws.skip[u.level] : ws.x[in.p1 == ws.x[0] ? 1 : 0];
    int rc;
    if (u.kind == M_DOWN || u.kind == M_UP)
      rc = launch_unet_resample(in.p1, dst, B, hi, wi, in.c1, u.kind == M_UP, st);
    else if (u.kind == M_RES)
      rc = run_res(prec, u, in, dst, ws, B, hi, wi, cond, cbs, st);
    else
      rc = run_attn(prec, u, in.p1, dst, ws, B, hi, wi, cond, cbs, st);
    y = dst;
    return rc ? rc : m->tap(u.tap, dst, (int64_t)B * ho * wo * C, st);
  });
  if (rc || (rc = launch_unet_patch_out(y, m->proj_out_w, m->proj_out_b, x, sigma, sd, out, B, c.in_channels, H, W, c.patch_size, C0, st)))
    return rc;
  const int Kin = c.in_channels * c.patch_size * c.patch_size;
  return logvar ? launch_unet_logvar(y, m->proj_out_w + (size_t)Kin * C0, m->proj_out_b + Kin, logvar, B, h * w, C0, st) : 0;
}

// ------------------------------------------------------------------------------------------------
// training: the fp32 forward with a tape, then the reverse walk with every parameter's gradient
// ------------------------------------------------------------------------------------------------

// The training workspace: a forward's (UWs), the tape (patch_in's output, then every module's output: the input of the next), the stream
// gradient in two ping-pong buffers, each level's skip gradient, the backward's scratch, the conditioning's gradients, the reduction partials.
struct TWs {
  UWs f;
  std::vector<float*> tape;
  float *g[2] = {}, *gskip[KDB_MAX_LEVELS] = {};
  float *ga = nullptr, *gb = nullptr, *dqkv = nullptr, *stats = nullptr;
  float *dss = nullptr, *dcond = nullptr, *dwcat = nullptr, *dbcat = nullptr, *U = nullptr, *xin = nullptr, *part = nullptr;
  UNetMapGrad mg{};
  size_t total = 0;
};

// the input (sources, grid) of every module of m->mods, as unet_forward with a tape feeds it (M_CONCAT: unused)
struct ModIO {
  Src in;
  int h = 0, w = 0;
};

void carve_train(const KdbUNet* m, int B, int H, int W, void* workspace, TWs& t) {
  const KdbUNetConfig& c = m->cfg;
  carve(c, B, H, W, workspace, t.f);
  Carver cv(workspace ? static_cast<char*>(workspace) + t.f.total : nullptr, 256);
  auto take = [&](size_t floats) { return cv.take<float>(floats * sizeof(float)); };
  const int s0 = c.skip_stages, mw = c.mapping_out, A = m->ada_total, p = c.patch_size;
  const int Kin = c.in_channels * p * p, Kout = Kin + (c.has_variance ? 1 : 0);
  int h, w;
  level_dims(c, H, W, s0, &h, &w);
  const size_t M0 = (size_t)B * h * w;
  t.tape.assign(m->mods.size() + 1, nullptr);
  t.tape[0] = take(M0 * c.channels[std::max(0, s0 - 1)]);
  size_t elems = 0, stats = 0;
  walk(m, H, W, t.tape[0], [&](size_t i, const UMod& u, const Src& in, int hi, int wi, int ho, int wo, int C, float*& dst) {
    dst = t.tape[i + 1] = take((size_t)B * ho * wo * C);
    elems = std::max({elems, (size_t)B * hi * wi * (in.c1 + in.c2), (size_t)B * ho * wo * C, (size_t)B * hi * wi * 3 * u.c_out});
    if (u.kind == M_ATTN) stats = std::max(stats, (size_t)B * hi * wi * std::max(1, u.c_out / 64) * 3);
    return 0;
  });
  t.g[0] = take(elems);
  t.g[1] = take(elems);
  for (int l = s0; l < c.n_levels - 1; ++l) {
    int hl, wl;
    level_dims(c, H, W, l, &hl, &wl);
    t.gskip[l] = take((size_t)B * hl * wl * c.channels[l]);
  }
  t.ga = take(elems);
  t.gb = take(elems);
  t.dqkv = take(elems);
  t.stats = take(stats);
  t.dss = take((size_t)B * A);
  t.dcond = take((size_t)B * mw);
  t.dwcat = take((size_t)A * mw);
  t.dbcat = take((size_t)A);
  t.mg = UNetMapGrad{take((size_t)B * mw), take((size_t)B * mw), take((size_t)B * mw), take((size_t)B * mw), take((size_t)B * mw),
                     take((size_t)B * std::max(1, c.mapping_cond_dim))};
  t.U = take(M0 * Kout);
  t.xin = take(M0 * Kin);
  t.part = take((size_t)kTrainPartFloats);
  t.total = t.f.total + cv.total();
}

// The input-gradient weights of every convolution (launch_unet_flip_conv_weight of its tap-major copy), built by the first training call after
// a finalize into the model's kept allocations, in the order of mods
int ensure_bwd(KdbUNet* m, cudaStream_t st) {
  if (m->kept_ready) return 0;
  struct Flip { const float* src; int N, C, ks; const float** dst; };
  std::vector<Flip> flips;
  for (UMod& u : m->mods) {
    if (u.kind == M_RES) {
      flips.push_back({u.w1.f32, u.c_mid, u.c_in, 3, &u.w1t});
      flips.push_back({u.w2.f32, u.c_out, u.c_mid, 3, &u.w2t});
      if (u.skip_w.f32 != nullptr) flips.push_back({u.skip_w.f32, u.c_out, u.c_in, 1, &u.skip_t});
    } else if (u.kind == M_ATTN) {
      flips.push_back({u.w1.f32, 3 * u.c_out, u.c_out, 1, &u.w1t});
      flips.push_back({u.w2.f32, u.c_out, u.c_out, 1, &u.w2t});
    }
  }
  std::vector<size_t> floats;
  for (const Flip& f : flips) floats.push_back((size_t)f.N * f.C * f.ks * f.ks);
  if (int rc = m->keep(floats, "training call after a finalize builds the input-gradient weights", st)) return rc;
  for (size_t i = 0; i < flips.size(); ++i) {
    const Flip& f = flips[i];
    if (int rc = launch_unet_flip_conv_weight(f.src, m->kept[i], f.N, f.C, f.ks, st)) return rc;
    *f.dst = m->kept[i];
  }
  KDB_CUDA(cudaStreamSynchronize(st));
  m->kept_ready = true;
  return 0;
}

// The U-Net's refusal rule for a gradient buffer (check_grad): the buffers, and the blocks below skip_stages
int check_grad_key(const KdbUNet* m, const std::string& k) {
  const bool buffer = k == "timestep_embed.weight" || (k.size() >= 7 && k.compare(k.size() - 7, 7, ".kernel") == 0);
  KDB_REQUIRE(!buffer, KDB_ERR_BAD_ARG, "'%s' is a buffer, not a parameter", k.c_str());
  const KdbUNetConfig& c = m->cfg;
  for (int l = 0; l < c.skip_stages; ++l)   // the blocks of the levels below skip_stages, which the forward never runs
    for (const std::string& p : {"u_net.d_blocks." + std::to_string(l) + ".", "u_net.u_blocks." + std::to_string(c.n_levels - 1 - l) + "."})
      KDB_REQUIRE(k.compare(0, p.size(), p) != 0, KDB_ERR_BAD_ARG, "'%s' belongs to a block below skip_stages, which the forward never runs",
                  k.c_str());
  return 0;
}

ConvArgs conv_args(const float* in1, int c1, const float* in2, int c2, const float* w, const float* bias, float* out, int N, int B, int h, int wd) {
  ConvArgs a;
  a.in1 = in1, a.c1 = c1, a.in2 = in2, a.c2 = c2, a.w = w, a.bias = bias, a.out = out, a.N = N;
  a.B = B, a.H = h, a.W = wd;
  return a;
}

// ResConvBlock in reverse: g the gradient of its output [B, h, w, c_out]; writes that of its input, split as the input (out1: in.c1
// channels, out2: in.c2), the gradients of its weights and (into t.dss) those of its AdaGN mappers' outputs.  Recomputes n1 = gelu(AdaGN1(x)),
// h = conv1(n1) and n3 = gelu(AdaGN2(h)) with the forward's launches.
int res_vjp(KdbUNet* m, const UMod& u, const Src& in, const float* g, float* out1, float* out2, TWs& t, int B, int h, int w, const float* cond,
            int64_t cbs, cudaStream_t st) {
  UWs& ws = t.f;
  const int64_t M = (int64_t)B * h * w;
  const int A = m->ada_total;
  const std::string& p = u.prefix;
  int rc;
  if ((rc = launch_unet_adagn(in.p1, in.c1, in.p2, in.c2, ws.n1, cond, cbs, u.ada1, u.groups1, true, B, h * w, st)) ||
      (rc = launch_unet_conv(conv_args(ws.n1, u.c_in, nullptr, 0, u.w1.f32, u.b1, ws.n2, u.c_mid, B, h, w), 3, st)) ||
      (rc = launch_unet_adagn(ws.n2, u.c_mid, nullptr, 0, ws.qkv, cond, cbs, u.ada2, u.groups2, true, B, h * w, st)))
    return rc;
  // conv2: weight and bias gradients, then the gradient of n3 and through AdaGN2 + GELU that of h
  if ((rc = launch_wgrad_conv(g, u.c_out, ws.qkv, u.c_mid, nullptr, 0, m->grad(p + "main.6.weight"), B, h, w, 3, t.part, st)) ||
      (rc = launch_colsum(g, M, u.c_out, m->grad(p + "main.6.bias"), t.part, st)) ||
      (rc = launch_unet_conv(conv_args(g, u.c_out, nullptr, 0, u.w2t, nullptr, t.ga, u.c_mid, B, h, w), 3, st)) ||
      (rc = launch_unet_adagn_vjp(ws.n2, u.c_mid, nullptr, 0, t.ga, nullptr, t.gb, nullptr, cond, cbs, u.ada2, t.dss, A, u.groups2, true, B, h * w,
                                  st)))
    return rc;
  // conv1, then the gradient of n1
  if ((rc = launch_wgrad_conv(t.gb, u.c_mid, ws.n1, u.c_in, nullptr, 0, m->grad(p + "main.2.weight"), B, h, w, 3, t.part, st)) ||
      (rc = launch_colsum(t.gb, M, u.c_mid, m->grad(p + "main.2.bias"), t.part, st)) ||
      (rc = launch_unet_conv(conv_args(t.gb, u.c_mid, nullptr, 0, u.w1t, nullptr, t.ga, u.c_in, B, h, w), 3, st)))
    return rc;
  // the skip path's gradient (the 1x1 conv's input gradient, or g itself) is added by AdaGN1's backward
  const float* add = g;
  if (u.skip_t != nullptr) {
    if ((rc = launch_wgrad_conv(g, u.c_out, in.p1, in.c1, in.p2, in.c2, m->grad(p + "skip.weight"), B, h, w, 1, t.part, st)) ||
        (rc = launch_unet_conv(conv_args(g, u.c_out, nullptr, 0, u.skip_t, nullptr, t.gb, u.c_in, B, h, w), 1, st)))
      return rc;
    add = t.gb;
  }
  return launch_unet_adagn_vjp(in.p1, in.c1, in.p2, in.c2, t.ga, add, out1, out2, cond, cbs, u.ada1, t.dss, A, u.groups1, true, B, h * w, st);
}

// SelfAttention2d in reverse (x + out_proj(attn(qkv_proj(AdaGN(x))))), as res_vjp.  qkv_proj's q rows carry the folded softmax scale, so
// the gradients of its unfolded weight and bias rows are those of the folded ones times the scale.
int attn_vjp(KdbUNet* m, const UMod& u, const float* x, const float* g, float* out, TWs& t, int B, int h, int w, const float* cond, int64_t cbs,
             cudaStream_t st) {
  UWs& ws = t.f;
  const int64_t M = (int64_t)B * h * w;
  const int C = u.c_out, nh = std::max(1, C / 64);
  const float scale = 1.f / std::sqrt((float)(C / nh));
  const std::string& p = u.prefix;
  float *dwq = m->grad(p + "qkv_proj.weight"), *dbq = m->grad(p + "qkv_proj.bias");
  int rc;
  if ((rc = launch_unet_adagn(x, C, nullptr, 0, ws.n1, cond, cbs, u.ada1, u.groups1, false, B, h * w, st)) ||
      (rc = launch_unet_conv(conv_args(ws.n1, C, nullptr, 0, u.w1.f32, u.b1, ws.qkv, 3 * C, B, h, w), 1, st)) ||
      (rc = launch_attention_generic<float>(ws.qkv, ws.ao, B, h, w, nh, C / nh, KDB_ATTN_GLOBAL, 0, 0, st)))
    return rc;
  if ((rc = launch_wgrad_conv(g, C, ws.ao, C, nullptr, 0, m->grad(p + "out_proj.weight"), B, h, w, 1, t.part, st)) ||
      (rc = launch_colsum(g, M, C, m->grad(p + "out_proj.bias"), t.part, st)) ||
      (rc = launch_unet_conv(conv_args(g, C, nullptr, 0, u.w2t, nullptr, t.ga, C, B, h, w), 1, st)) ||
      (rc = launch_attention_vjp(ws.qkv, ws.ao, t.ga, t.dqkv, t.stats, B, h, w, nh, C / nh, KDB_ATTN_GLOBAL, 0, 0, st)))
    return rc;
  if ((rc = launch_wgrad_conv(t.dqkv, 3 * C, ws.n1, C, nullptr, 0, dwq, B, h, w, 1, t.part, st)) ||
      (rc = launch_colsum(t.dqkv, M, 3 * C, dbq, t.part, st)) || (rc = launch_unet_scale(dwq, (int64_t)C * C, scale, st)) ||
      (rc = launch_unet_scale(dbq, C, scale, st)) ||
      (rc = launch_unet_conv(conv_args(t.dqkv, 3 * C, nullptr, 0, u.w1t, nullptr, t.ga, C, B, h, w), 1, st)))
    return rc;
  return launch_unet_adagn_vjp(x, C, nullptr, 0, t.ga, g, out, nullptr, cond, cbs, u.ada1, t.dss, m->ada_total, u.groups1, false, B, h * w, st);
}

// out = the fp32 forward of F (bit for bit unet_forward's launches, writing the tape), then u^T dF/dparam + dlogvar^T dlogvar/dparam for every
// bound parameter by a walk of the modules in reverse: proj_out, the UBlocks (innermost last), the DBlocks, proj_in; then the AdaGN mappers and
// the mapping network.  dlogvar == nullptr: the logvar term is absent.
int unet_train(KdbUNet* m, int B, int H, int W, const float* x, const float* sigma, const float* aug, const float* mcond, const float* cond,
               int64_t cbs, const float* u, const float* dlogvar, float* out, TWs& t, cudaStream_t st) {
  const KdbUNetConfig& c = m->cfg;
  int rc = ensure_bwd(m, st);
  if (rc || (rc = unet_forward(m, KDB_PREC_FP32, B, H, W, x, sigma, 0.f, cond, cbs, out, t.f, st, t.tape.data()))) return rc;
  const int s0 = c.skip_stages, C0 = c.channels[std::max(0, s0 - 1)], p = c.patch_size;
  const int Kin = c.in_channels * p * p, Kout = Kin + (c.has_variance ? 1 : 0);
  int h, w;
  level_dims(c, H, W, s0, &h, &w);
  const int64_t M0 = (int64_t)B * h * w;
  float* part = t.part;
  // proj_out + pixel_shuffle: U = the patch rows of u, with a column for the variance channel the output drops: dlogvar[b] / T on image b's
  // T tokens (logvar[b] is their mean), or zero
  if ((rc = launch_unet_unshuffle(u, t.U, B, c.in_channels, H, W, p, Kout, dlogvar, st)) ||
      (rc = launch_wgrad(t.U, Kout, t.tape.back(), C0, m->grad("proj_out.weight"), M0, Kout, C0, part, st)) ||
      (rc = launch_colsum(t.U, M0, Kout, m->grad("proj_out.bias"), part, st)) ||
      (rc = launch_unet_proj_out_vjp(t.U, m->proj_out_w, t.g[0], M0, Kout, C0, st)))
    return rc;
  std::vector<ModIO> io(m->mods.size());
  walk(m, H, W, t.tape[0], [&](size_t i, const UMod&, const Src& in, int hi, int wi, int, int, int, float*& dst) {
    io[i] = ModIO{in, hi, wi};
    dst = t.tape[i + 1];
    return 0;
  });
  int gi = 0;   // t.g[gi]: the gradient of the output of the module being reversed
  for (size_t k = m->mods.size(); k-- > 0;) {
    const UMod& mod = m->mods[k];
    const ModIO& q = io[k];
    float *g = t.g[gi], *gin = t.g[gi ^ 1];
    switch (mod.kind) {
      case M_CONCAT:
        continue;
      case M_DOWN:   // its input is the previous level's DBlock output, which the UBlock of that level also read: add that skip gradient
        rc = launch_unet_resample_vjp(g, t.gskip[mod.level - 1], gin, B, q.h, q.w, q.in.c1, false, st);
        break;
      case M_UP:
        rc = launch_unet_resample_vjp(g, nullptr, gin, B, q.h, q.w, q.in.c1, true, st);
        break;
      case M_RES:
        rc = res_vjp(m, mod, q.in, g, gin, q.in.p2 ? t.gskip[mod.level] : nullptr, t, B, q.h, q.w, cond, cbs, st);
        break;
      default:
        rc = attn_vjp(m, mod, q.in.p1, g, gin, t, B, q.h, q.w, cond, cbs, st);
    }
    if (rc) return rc;
    gi ^= 1;
  }
  // proj_in: its input is the pixel_unshuffle of x (the caller's c_in-scaled input)
  if ((rc = launch_unet_unshuffle(x, t.xin, B, c.in_channels, H, W, p, Kin, nullptr, st)) ||
      (rc = launch_wgrad(t.g[gi], C0, t.xin, Kin, m->grad("proj_in.weight"), M0, C0, Kin, part, st)) ||
      (rc = launch_colsum(t.g[gi], M0, C0, m->grad("proj_in.bias"), part, st)))
    return rc;
  // the AdaGN mappers, concatenated as at finalize: one weight gradient over the B conditioning rows, scattered to the bound keys; then the
  // gradient of the mapping network's output and its backward
  const int A = m->ada_total, mw = c.mapping_out, mcd = c.mapping_cond_dim;
  if ((rc = launch_wgrad(t.dss, A, cond + A, cbs, t.dwcat, B, A, mw, part, st)) || (rc = launch_colsum(t.dss, B, A, t.dbcat, part, st))) return rc;
  for (const UMod& mod : m->mods) {
    const int n_ada = mod.kind == M_RES ? 2 : (mod.kind == M_ATTN ? 1 : 0);
    for (int i = 0; i < n_ada; ++i) {
      const int off = i ? mod.ada2 : mod.ada1, C = i ? mod.c_mid : (mod.kind == M_RES ? mod.c_in : mod.c_out);
      const std::string key = mod.prefix + (mod.kind == M_ATTN ? "norm_in." : i ? "main.4." : "main.0.");
      if (float* dw = m->grad(key + "mapper.weight"))
        KDB_CUDA(cudaMemcpyAsync(dw, t.dwcat + (size_t)off * mw, sizeof(float) * 2 * C * mw, cudaMemcpyDeviceToDevice, st));
      if (float* db = m->grad(key + "mapper.bias"))
        KDB_CUDA(cudaMemcpyAsync(db, t.dbcat + off, sizeof(float) * 2 * C, cudaMemcpyDeviceToDevice, st));
    }
  }
  const UNetMapGrad& mg = t.mg;
  if ((rc = launch_gemm_vjp(t.dss, m->cw.ada_w, t.dcond, B, A, mw, VJP_STORE, 0, 0, 0, st)) ||
      (rc = launch_unet_mapping_vjp(m->cw, B, sigma, aug, mcond, t.dcond, mg, st)) ||
      (rc = launch_wgrad(mg.dz1, mw, mg.a0, mw, m->grad("mapping.2.weight"), B, mw, mw, part, st)) ||
      (rc = launch_colsum(mg.dz1, B, mw, m->grad("mapping.2.bias"), part, st)) ||
      (rc = launch_wgrad(mg.dz0, mw, mg.h0, mw, m->grad("mapping.0.weight"), B, mw, mw, part, st)) ||
      (rc = launch_colsum(mg.dz0, B, mw, m->grad("mapping.0.bias"), part, st)))
    return rc;
  return mcd > 0 ? launch_wgrad(mg.dh0, mw, mg.v, mcd, m->grad("mapping_cond.weight"), B, mw, mcd, part, st) : 0;
}

// the grid checks of kdb_unet_forward and kdb_unet_forward_train
int check_grid(const KdbUNetConfig& c, const char* what, int height, int width) {
  KDB_REQUIRE(height > 0 && width > 0 && height % c.patch_size == 0 && width % c.patch_size == 0, KDB_ERR_BAD_SHAPE,
              "%s: %dx%d not divisible by the patch size %d", what, height, width, c.patch_size);
  for (int l = c.skip_stages; l < c.n_levels; ++l) {
    int h, w;
    level_dims(c, height, width, l, &h, &w);
    const bool down_from = l < c.n_levels - 1;        // this grid is downsampled, and the upsample must restore it
    KDB_REQUIRE(h >= 2 && w >= 2 && (!down_from || (h % 2 == 0 && w % 2 == 0)), KDB_ERR_BAD_SHAPE,
                "%s: level %d grid %dx%d (every level but the innermost needs an even grid, every level >= 2x2)", what, l, h, w);
  }
  return 0;
}

// the aug_cond / mapping_cond checks of kdb_unet_conditioning, kdb_unet_forward_train and kdb_unet_mapping_vjp
int check_conds(const KdbUNetConfig& c, const char* what, const float* aug_cond, const float* mapping_cond) {
  KDB_REQUIRE(!(aug_cond && !c.augment_wrapper), KDB_ERR_BAD_ARG, "%s: aug_cond needs the augment wrapper", what);
  KDB_REQUIRE(!(c.augment_wrapper && c.mapping_cond_dim > 9 && mapping_cond == nullptr), KDB_ERR_BAD_ARG,
              "%s: mapping_cond must be given (mapping_cond_dim %d)", what, c.mapping_cond_dim - 9);
  KDB_REQUIRE(!(mapping_cond && c.mapping_cond_dim == (c.augment_wrapper ? 9 : 0)), KDB_ERR_BAD_ARG, "%s: the model takes no mapping_cond", what);
  return 0;
}

// kdb_unet_forward and kdb_unet_forward_variance (logvar != nullptr); `what` names the entry point in errors
int forward_entry(KdbUNet* m, const char* what, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                  const float* cond, int64_t cond_batch_stride, float* out, float* logvar, void* workspace, size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "%s: model NULL or not finalized", what);
  KDB_REQUIRE(x && sigma && cond && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "%s: NULL argument", what);
  KDB_REQUIRE(precision == KDB_PREC_FP32 || precision == KDB_PREC_TF32 || precision == KDB_PREC_FP16, KDB_ERR_UNSUPPORTED,
              "%s: the fp32, tf32 and fp16 paths are built (precision %d)", what, precision);
  const KdbUNetConfig& c = m->cfg;
  if (int rc = check_grid(c, what, height, width)) return rc;
  UWs ws;
  carve(c, batch, height, width, workspace, ws);
  KDB_REQUIRE(ws.total <= workspace_bytes, KDB_ERR_WORKSPACE, "%s: workspace %zu < required %zu", what, workspace_bytes, ws.total);
  return m->disarm_tap(unet_forward(m, precision, batch, height, width, x, sigma, sigma_data, cond, cond_batch_stride, out, ws, (cudaStream_t)stream,
                                    nullptr, logvar));
}

// kdb_unet_forward_train and kdb_unet_forward_train_variance (dlogvar != nullptr)
int train_entry(KdbUNet* m, const char* what, int precision, int batch, int height, int width, const float* x, const float* sigma, const float* aug_cond,
                const float* mapping_cond, const float* cond, int64_t cond_batch_stride, const float* cotangent, const float* dlogvar, float* out,
                void* workspace, size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m, KDB_ERR_BAD_ARG, "%s: NULL model", what);
  KDB_REQUIRE(precision == KDB_PREC_FP32, KDB_ERR_UNSUPPORTED, "%s: U-Net training runs at fp32 (precision %d)", what, precision);
  KDB_REQUIRE(m->finalized, KDB_ERR_NOT_FINAL, "%s: model not finalized", what);
  KDB_REQUIRE(x && sigma && cond && cotangent && out && workspace && batch > 0, KDB_ERR_BAD_ARG, "%s: NULL argument", what);
  const KdbUNetConfig& c = m->cfg;
  int rc;
  if ((rc = check_conds(c, what, aug_cond, mapping_cond))) return rc;
  if ((rc = check_train(m, what, cond_batch_stride, kdb_unet_cond_stride(m), check_grad_key))) return rc;
  if ((rc = check_grid(c, what, height, width))) return rc;
  TWs t;
  carve_train(m, batch, height, width, workspace, t);
  KDB_REQUIRE(t.total <= workspace_bytes, KDB_ERR_WORKSPACE, "%s: workspace %zu < required %zu", what, workspace_bytes, t.total);
  return m->disarm_tap(unet_train(m, batch, height, width, x, sigma, aug_cond, mapping_cond, cond, cond_batch_stride, cotangent, dlogvar, out, t,
                                  (cudaStream_t)stream));
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
  m->kept_ready = false;
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
  if (int rc = check_conds(m->cfg, "unet_conditioning", aug_cond, mapping_cond)) return rc;
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
  return forward_entry(m, "unet_forward", precision, batch, height, width, x, sigma, sigma_data, cond, cond_batch_stride, out, nullptr, workspace,
                       workspace_bytes, stream);
}

int kdb_unet_forward_variance(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma, float sigma_data,
                              const float* cond, int64_t cond_batch_stride, float* out, float* logvar, void* workspace, size_t workspace_bytes,
                              void* stream) {
  KDB_REQUIRE(m && m->cfg.has_variance, KDB_ERR_BAD_ARG, "unet_forward_variance: model NULL or without has_variance");
  KDB_REQUIRE(logvar, KDB_ERR_BAD_ARG, "unet_forward_variance: NULL logvar");
  return forward_entry(m, "unet_forward_variance", precision, batch, height, width, x, sigma, sigma_data, cond, cond_batch_stride, out, logvar,
                       workspace, workspace_bytes, stream);
}

int kdb_unet_set_grad(KdbUNet* m, const char* key, float* data, const int64_t* shape, int ndim) {
  return set_grad(m, "unet_set_grad", key, data, shape, ndim, check_grad_key);
}

int64_t kdb_unet_train_workspace_bytes(const KdbUNet* m, int batch, int height, int width) {
  KDB_REQUIRE(m && batch > 0 && height > 0 && width > 0, KDB_ERR_BAD_ARG, "unet_train_workspace_bytes: bad argument");
  KDB_REQUIRE(m->finalized, KDB_ERR_NOT_FINAL, "unet_train_workspace_bytes: model not finalized");
  TWs t;
  carve_train(m, batch, height, width, nullptr, t);
  return (int64_t)t.total;
}

int kdb_unet_forward_train(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma, const float* aug_cond,
                           const float* mapping_cond, const float* cond, int64_t cond_batch_stride, const float* cotangent, float* out,
                           void* workspace, size_t workspace_bytes, void* stream) {
  return train_entry(m, "unet_forward_train", precision, batch, height, width, x, sigma, aug_cond, mapping_cond, cond, cond_batch_stride, cotangent,
                     nullptr, out, workspace, workspace_bytes, stream);
}

int kdb_unet_forward_train_variance(KdbUNet* m, int precision, int batch, int height, int width, const float* x, const float* sigma,
                                    const float* aug_cond, const float* mapping_cond, const float* cond, int64_t cond_batch_stride,
                                    const float* cotangent, const float* dlogvar, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  KDB_REQUIRE(m && m->cfg.has_variance, KDB_ERR_BAD_ARG, "unet_forward_train_variance: model NULL or without has_variance");
  KDB_REQUIRE(dlogvar, KDB_ERR_BAD_ARG, "unet_forward_train_variance: NULL dlogvar");
  return train_entry(m, "unet_forward_train_variance", precision, batch, height, width, x, sigma, aug_cond, mapping_cond, cond, cond_batch_stride,
                     cotangent, dlogvar, out, workspace, workspace_bytes, stream);
}

int kdb_unet_conv_wgrad(const float* dy, int n_out, const float* in1, int c1, const float* in2, int c2, float* dw, int batch, int h, int w, int ksize,
                        float* scratch, void* stream) {
  KDB_REQUIRE(dy && in1 && dw && scratch && n_out > 0 && c1 > 0 && c2 >= 0 && (c2 == 0 || in2) && batch > 0 && h > 0 && w > 0, KDB_ERR_BAD_ARG,
              "unet_conv_wgrad: bad argument");
  KDB_REQUIRE(ksize == 1 || ksize == 3, KDB_ERR_BAD_ARG, "unet_conv_wgrad: kernel size %d", ksize);
  return launch_wgrad_conv(dy, n_out, in1, c1, in2, c2, dw, batch, h, w, ksize, scratch, (cudaStream_t)stream);
}

int kdb_unet_adagn_vjp(const float* in1, int c1, const float* in2, int c2, const float* dy, const float* add, float* dx1, float* dx2,
                       const float* cond, int64_t cond_batch_stride, int ada_off, float* dcond, int64_t dcond_batch_stride, int groups, int gelu,
                       int batch, int hw, void* stream) {
  KDB_REQUIRE(in1 && dy && dx1 && cond && dcond && c1 > 0 && c2 >= 0 && batch > 0 && hw > 0 && ada_off >= 0, KDB_ERR_BAD_ARG,
              "unet_adagn_vjp: bad argument");
  return launch_unet_adagn_vjp(in1, c1, in2, c2, dy, add, dx1, dx2, cond, cond_batch_stride, ada_off, dcond, dcond_batch_stride, groups, gelu != 0,
                               batch, hw, (cudaStream_t)stream);
}

int kdb_unet_flip_conv_weight(const float* w_tapmajor, float* out, int n_out, int c_in, int ksize, void* stream) {
  KDB_REQUIRE(w_tapmajor && out && n_out > 0 && c_in > 0 && (ksize == 1 || ksize == 3), KDB_ERR_BAD_ARG, "unet_flip_conv_weight: bad argument");
  return launch_unet_flip_conv_weight(w_tapmajor, out, n_out, c_in, ksize, (cudaStream_t)stream);
}

int kdb_unet_resample_vjp(const float* dout, const float* add, float* din, int batch, int h, int w, int c, int up, void* stream) {
  KDB_REQUIRE(dout && din && batch > 0 && c > 0, KDB_ERR_BAD_ARG, "unet_resample_vjp: bad argument");
  return launch_unet_resample_vjp(dout, add, din, batch, h, w, c, up != 0, (cudaStream_t)stream);
}

int kdb_unet_mapping_vjp(const KdbUNet* m, int rows, const float* sigma, const float* aug_cond, const float* mapping_cond, const float* dcond,
                         float* h0, float* a0, float* dz0, float* dz1, float* dh0, float* v, void* stream) {
  KDB_REQUIRE(m && m->finalized, KDB_ERR_NOT_FINAL, "unet_mapping_vjp: model NULL or not finalized");
  KDB_REQUIRE(rows > 0 && sigma && dcond && h0 && a0 && dz0 && dz1 && dh0 && (v || m->cfg.mapping_cond_dim == 0), KDB_ERR_BAD_ARG,
              "unet_mapping_vjp: bad argument");
  if (int rc = check_conds(m->cfg, "unet_mapping_vjp", aug_cond, mapping_cond)) return rc;
  return launch_unet_mapping_vjp(m->cw, rows, sigma, aug_cond, mapping_cond, dcond, UNetMapGrad{h0, a0, dz0, dz1, dh0, v}, (cudaStream_t)stream);
}

int kdb_unet_proj_out_vjp(const float* u, const float* w, float* out, int64_t rows, int n, int k, void* stream) {
  KDB_REQUIRE(u && w && out && rows > 0 && n > 0 && k > 0, KDB_ERR_BAD_ARG, "unet_proj_out_vjp: bad argument");
  return launch_unet_proj_out_vjp(u, w, out, rows, n, k, (cudaStream_t)stream);
}

int kdb_unet_unshuffle(const float* x, float* out, int batch, int c, int h, int w, int p, int ld, void* stream) {
  KDB_REQUIRE(x && out && batch > 0 && c > 0 && p > 0 && h > 0 && w > 0 && h % p == 0 && w % p == 0 && ld >= c * p * p, KDB_ERR_BAD_ARG,
              "unet_unshuffle: bad argument");
  return launch_unet_unshuffle(x, out, batch, c, h, w, p, ld, nullptr, (cudaStream_t)stream);
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
