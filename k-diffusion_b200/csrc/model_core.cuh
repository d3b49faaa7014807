// model_core.cuh -- host-side state every model engine shares (engine.cu, unet_engine.cu): the borrowed state-dict tensors and their
// shape-checked lookup, owned device allocations, the debug tap, and the carver that lays out a caller's workspace.
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
  bool finalized = false;
  std::vector<void*> owned;
  // debug tap: armed by kdb_*_debug_tap, filled by the forward's tap() at the stage of that name, disarmed when the forward returns
  std::string tap_name;
  float* tap_out = nullptr;
  int64_t tap_cap = 0, tap_count = 0;

  ~ModelCore() { free_all(); }

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
