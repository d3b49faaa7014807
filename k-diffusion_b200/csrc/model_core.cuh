// model_core.cuh -- host-side state every model engine shares (engine.cu, unet_engine.cu): the borrowed state-dict tensors and their
// shape-checked lookup, the bound gradient buffers, owned device allocations and the derived copies kept across finalizes, the debug
// tap, and the carver that lays out a caller's workspace.
#pragma once
#include <initializer_list>
#include <string>
#include <unordered_map>
#include <vector>

#include "model_kernels.cuh"

namespace kdb {

struct ModelCore {
  struct TensorRef {
    const float* p = nullptr;
    std::vector<int64_t> shape;
  };
  std::unordered_map<std::string, TensorRef> tensors;
  std::unordered_map<std::string, TensorRef> grads;   // kdb_*_set_grad: gradient buffers by state-dict key (written: p is not const)
  bool finalized = false;
  std::vector<void*> owned;
  // The derived weight copies a training call builds (ensure_tf32, ensure_bwd), one allocation per copy in the order of its list, kept
  // across finalizes instead of in `owned`.  Separate allocations, not one buffer: with one buffer, kdb_model_finalize's reallocation of
  // the owned buffers took ~13 ms instead of ~5.5 ms per rebind on cfg1 (H100 80GB HBM3, 700 W), which made every tf32 training step
  // that much slower
  std::vector<float*> kept;
  bool kept_ready = false;   // the kept copies are of the weights the last finalize read
  // debug tap: armed by kdb_*_debug_tap, filled by the forward's tap() at the stage of that name, disarmed when the forward returns
  std::string tap_name;
  float* tap_out = nullptr;
  int64_t tap_cap = 0, tap_count = 0;

  ~ModelCore() {
    free_all();
    for (float* p : kept) cudaFree(p);
  }

  // the registered tensor `key`, which must have shape `want`
  int get(const std::string& key, std::initializer_list<int64_t> want, const float** out) const {
    auto it = tensors.find(key);
    if (it == tensors.end()) {
      set_error("missing state-dict entry '%s'", key.c_str());
      return KDB_ERR_MISSING_KEY;
    }
    if (it->second.shape != std::vector<int64_t>(want)) {
      std::string got, exp;
      for (auto v : it->second.shape) got += std::to_string(v) + ",";
      for (auto v : want) exp += std::to_string(v) + ",";
      set_error("shape mismatch for '%s': got [%s] expected [%s]", key.c_str(), got.c_str(), exp.c_str());
      return KDB_ERR_BAD_SHAPE;
    }
    *out = it->second.p;
    return 0;
  }

  // `count` elements of device memory owned (and freed) by the model, with slack past the end for vector loads
  template <typename T>
  int alloc(T** p, size_t count) {
    void* q = nullptr;
    KDB_CUDA(cudaMalloc(&q, count * sizeof(T) + 1024));
    owned.push_back(q);
    *p = reinterpret_cast<T*>(q);
    return 0;
  }

  void free_all() {
    for (void* p : owned) cudaFree(p);
    owned.clear();
  }

  // The first build of the kept copies after a finalize, whose allocations hold floats[i] floats each: refused under CUDA-graph capture
  // (`what`: the call and what it builds), and `kept` grown to them once per handle (the shapes are the config's)
  int keep(const std::vector<size_t>& floats, const char* what, cudaStream_t st) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    KDB_CUDA(cudaStreamIsCapturing(st, &cs));
    KDB_REQUIRE(cs == cudaStreamCaptureStatusNone, KDB_ERR_UNSUPPORTED, "the first %s: it must run outside CUDA-graph capture", what);
    while (kept.size() < floats.size()) {
      void* p = nullptr;
      KDB_CUDA(cudaMalloc(&p, sizeof(float) * floats[kept.size()] + 1024));
      kept.push_back(static_cast<float*>(p));
    }
    return 0;
  }

  // the gradient buffer bound to `key`, or nullptr
  float* grad(const std::string& key) const {
    auto it = grads.find(key);
    return it == grads.end() ? nullptr : const_cast<float*>(it->second.p);
  }

  // copies the n elements at p to the armed tap buffer as fp32 when `name` is the armed stage (tap_count < 0: the buffer is too short)
  template <typename T>
  int tap(const std::string& name, const T* p, int64_t n, cudaStream_t st) {
    if (!tapped(name)) return 0;
    if (n > tap_cap) {
      tap_count = -n;
      return 0;
    }
    tap_count = n;
    return launch_to_f32<T>(p, tap_out, n, st);
  }
  bool tapped(const std::string& name) const { return tap_out != nullptr && tap_name == name; }

  // the end of every forward: disarms the tap and passes the forward's return code through
  int disarm_tap(int rc) {
    tap_out = nullptr;
    tap_name.clear();
    return rc;
  }
};

// GET(key, &ptr, dims...): looks up `key` with shape {dims...} in the model `m` of the enclosing function, returning on failure
#define GET(key, out, ...)                          \
  do {                                              \
    int rc__ = m->get((key), {__VA_ARGS__}, (out)); \
    if (rc__) return rc__;                          \
  } while (0)

// the kdb_*_set_tensor and kdb_*_debug_tap entry points of every engine
inline int set_tensor(ModelCore* m, const char* key, const float* data, const int64_t* shape, int ndim) {
  KDB_REQUIRE(m && key && data && ndim >= 0 && ndim <= 4 && (ndim == 0 || shape), KDB_ERR_BAD_ARG, "set_tensor: bad argument");
  ModelCore::TensorRef& t = m->tensors[key];
  t.p = data;
  t.shape.assign(shape, shape + ndim);
  m->finalized = false;
  return 0;
}

inline int arm_tap(ModelCore* m, const char* name, float* out, int64_t capacity) {
  KDB_REQUIRE(m && name && out && capacity > 0, KDB_ERR_BAD_ARG, "debug_tap: bad argument");
  m->tap_name = name;
  m->tap_out = out;
  m->tap_cap = capacity;
  m->tap_count = 0;
  return 0;
}

// A gradient buffer for `k` is refused unless the model has a tensor of that key and shape, and then by the engine's `rule` (the tensors
// that are no parameter its training call writes)
template <typename M>
int check_grad(const M* m, const std::string& k, const std::vector<int64_t>& shape, int (*rule)(const M*, const std::string&)) {
  auto it = m->tensors.find(k);
  KDB_REQUIRE(it != m->tensors.end(), KDB_ERR_MISSING_KEY, "gradient bound to '%s', which is no tensor of the model", k.c_str());
  KDB_REQUIRE(it->second.shape == shape, KDB_ERR_BAD_SHAPE, "gradient of '%s' has the wrong shape", k.c_str());
  return rule(m, k);
}

// the kdb_*_set_grad entry points of every engine (data == nullptr unbinds `key`)
template <typename M>
int set_grad(M* m, const char* what, const char* key, float* data, const int64_t* shape, int ndim, int (*rule)(const M*, const std::string&)) {
  KDB_REQUIRE(m && key && ndim >= 0 && ndim <= 4 && (ndim == 0 || shape), KDB_ERR_BAD_ARG, "%s: bad argument", what);
  if (data == nullptr) {
    m->grads.erase(key);
    return 0;
  }
  std::vector<int64_t> dims(shape, shape + ndim);
  if (int rc = check_grad(m, key, dims, rule)) return rc;
  m->grads[key] = ModelCore::TensorRef{data, dims};
  return 0;
}

// the binding checks of every kdb_*_forward_train: one conditioning row per image, and every bound gradient again (the weights may have
// been rebound since the gradients were)
template <typename M>
int check_train(const M* m, const char* what, int64_t cond_batch_stride, int64_t cond_stride, int (*rule)(const M*, const std::string&)) {
  KDB_REQUIRE(cond_batch_stride == cond_stride, KDB_ERR_BAD_ARG,
              "%s: one conditioning row per image (cond_batch_stride %lld, the row stride is %lld)", what, (long long)cond_batch_stride,
              (long long)cond_stride);
  for (const auto& kv : m->grads)
    if (int rc = check_grad(m, kv.first, kv.second.shape, rule)) return rc;
  return 0;
}

// Lays consecutive buffers out in a workspace, each starting `align` bytes apart; the workspace's own start is rounded up to `align`,
// and with workspace == nullptr the carver only sizes.  total(): the bytes a caller must pass, the alignment slack included.
struct Carver {
  char* base;
  size_t align, off = 0;
  Carver(void* workspace, size_t align_)
      : base(workspace ? reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(workspace), align_)) : nullptr), align(align_) {}
  template <typename T = char>
  T* take(size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes, align);
    return reinterpret_cast<T*>(p);
  }
  size_t total() const { return off + align; }
};

}  // namespace kdb
