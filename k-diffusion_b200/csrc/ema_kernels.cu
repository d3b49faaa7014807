// ema_kernels.cu -- kdb_ema_update: the exponential moving average of a model's parameters and the copy of its buffers after each
// optimizer step (reference utils.py ema_update: one lerp_ per parameter, one copy_ per buffer) in one launch.
// Every element is written by one thread, no atomics.  The lerp is torch's CUDA lerp with a scalar weight, written with explicit
// roundings so that the compiler's FMA contraction cannot change it: bit for bit what lerp_ gives on the same GPU.
#include <algorithm>
#include <map>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace kdb {

namespace {

constexpr int kEmaThreads = 256;
constexpr int kEmaUnroll = 4;                                   // independent 128-bit loads in flight per thread and operand
constexpr int64_t kEmaChunkQuads = kEmaThreads * kEmaUnroll;    // groups of four elements per CTA work item

// A segment as the kernel walks it: `head` scalar elements up to the first 16-byte boundary of dst, then `quads` groups of four (float4
// when src and dst are co-aligned, four scalars otherwise), then `tail` < 4 scalar elements.  Work item `chunk0 + k` is the k-th run of
// kEmaChunkQuads groups; item chunk0 also does the head and tail.
struct EmaSegDev {
  const float* src;
  float* dst;
  int64_t quads, chunk0;
  int head, tail, mode, vec;
};

// torch's lerp (ATen/native/Lerp.h) in fp32 with the weight's complement formed on the device as torch forms it, each branch one fused
// multiply-add as nvcc contracts it in torch's kernel: |w| < 0.5 ? self + w (end - self) : end - (end - self) (1 - w)
__device__ __forceinline__ float lerp_torch(float self, float end, float w, float one_minus_w) {
  const float d = __fsub_rn(end, self);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, d, self) : __fmaf_rn(-d, one_minus_w, end);
}

__device__ __forceinline__ void ema_one(const EmaSegDev& s, int64_t i, float w, float omw) {
  const float v = __ldg(s.src + i);
  s.dst[i] = s.mode == KDB_EMA_COPY ? v : lerp_torch(s.dst[i], v, w, omw);
}

__global__ void __launch_bounds__(kEmaThreads) ema_update_kernel(const EmaSegDev* __restrict__ segs, int n_segs, int64_t n_chunks, float w) {
  const float omw = __fsub_rn(1.f, w);
  for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    int lo = 0, hi = n_segs - 1;   // the last segment whose chunk0 <= c (every segment has at least one chunk)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (segs[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    const EmaSegDev s = segs[lo];
    const int64_t k = c - s.chunk0;
    if (k == 0) {
      if ((int)threadIdx.x < s.head) ema_one(s, threadIdx.x, w, omw);
      if ((int)threadIdx.x < s.tail) ema_one(s, s.head + 4 * s.quads + threadIdx.x, w, omw);
    }
    const int64_t q0 = k * kEmaChunkQuads, q1 = std::min(s.quads, q0 + kEmaChunkQuads);
    const float* src = s.src + s.head;
    float* dst = s.dst + s.head;
    if (s.vec) {
      float4 a[kEmaUnroll], b[kEmaUnroll];
#pragma unroll
      for (int u = 0; u < kEmaUnroll; ++u) {
        const int64_t q = q0 + u * kEmaThreads + threadIdx.x;
        if (q < q1) {
          a[u] = __ldg(reinterpret_cast<const float4*>(src) + q);
          if (s.mode != KDB_EMA_COPY) b[u] = reinterpret_cast<const float4*>(dst)[q];
        }
      }
#pragma unroll
      for (int u = 0; u < kEmaUnroll; ++u) {
        const int64_t q = q0 + u * kEmaThreads + threadIdx.x;
        if (q >= q1) continue;
        float4 o = a[u];
        if (s.mode != KDB_EMA_COPY) {
          o.x = lerp_torch(b[u].x, a[u].x, w, omw);
          o.y = lerp_torch(b[u].y, a[u].y, w, omw);
          o.z = lerp_torch(b[u].z, a[u].z, w, omw);
          o.w = lerp_torch(b[u].w, a[u].w, w, omw);
        }
        reinterpret_cast<float4*>(dst)[q] = o;
      }
    } else {
      for (int64_t q = q0 + threadIdx.x; q < q1; q += kEmaThreads)
#pragma unroll
        for (int e = 0; e < 4; ++e) ema_one(s, s.head + 4 * q + e, w, omw);
    }
  }
}

// The device copy of the segment table, per device: the caller's host table is expanded into a pinned staging buffer and copied to the
// device on the call's stream.  `copied` marks the end of that copy (the staging buffer may be rewritten after it), `done` the end of
// the kernel (a call on another stream waits for it before it overwrites the device table).
struct EmaTable {
  EmaSegDev* dev = nullptr;
  EmaSegDev* pinned = nullptr;
  size_t cap = 0;
  cudaEvent_t copied = nullptr, done = nullptr;
};
std::mutex g_ema_mutex;
std::map<int, EmaTable> g_ema_tables;

int ema_table(int device, size_t n, EmaTable*& out) {
  EmaTable& t = g_ema_tables[device];
  if (t.copied == nullptr) {
    KDB_CUDA(cudaEventCreateWithFlags(&t.copied, cudaEventDisableTiming));
    KDB_CUDA(cudaEventCreateWithFlags(&t.done, cudaEventDisableTiming));
  }
  if (t.cap < n) {
    const size_t cap = std::max(n, 2 * t.cap);
    KDB_CUDA(cudaEventSynchronize(t.done));
    if (t.dev) KDB_CUDA(cudaFree(t.dev));
    if (t.pinned) KDB_CUDA(cudaFreeHost(t.pinned));
    t.dev = nullptr;
    t.pinned = nullptr;
    t.cap = 0;
    KDB_CUDA(cudaMalloc(&t.dev, cap * sizeof(EmaSegDev)));
    KDB_CUDA(cudaMallocHost(&t.pinned, cap * sizeof(EmaSegDev)));
    t.cap = cap;
  }
  out = &t;
  return 0;
}

}  // namespace

}  // namespace kdb

using namespace kdb;

extern "C" {

int kdb_ema_update(const KdbEmaSeg* segs_host, int n_segs, float weight, void* stream) {
  KDB_REQUIRE(segs_host != nullptr, KDB_ERR_BAD_ARG, "ema_update: NULL segment table");
  KDB_REQUIRE(n_segs >= 0, KDB_ERR_BAD_ARG, "ema_update: %d segments", n_segs);
  std::vector<EmaSegDev> segs;
  segs.reserve(n_segs);
  int64_t chunks = 0;
  for (int i = 0; i < n_segs; ++i) {
    const KdbEmaSeg& g = segs_host[i];
    KDB_REQUIRE(g.mode == KDB_EMA_LERP || g.mode == KDB_EMA_COPY, KDB_ERR_BAD_ARG, "ema_update: segment %d has mode %d", i, (int)g.mode);
    KDB_REQUIRE(g.n >= 0, KDB_ERR_BAD_SHAPE, "ema_update: segment %d has %lld elements", i, (long long)g.n);
    if (g.n == 0) continue;
    KDB_REQUIRE(g.src != nullptr && g.dst != nullptr, KDB_ERR_BAD_ARG, "ema_update: segment %d of %lld elements has a NULL pointer", i,
                (long long)g.n);
    const uintptr_t s = reinterpret_cast<uintptr_t>(g.src), d = reinterpret_cast<uintptr_t>(g.dst);
    KDB_REQUIRE(((s | d) & 3u) == 0, KDB_ERR_BAD_ARG, "ema_update: segment %d is not 4-byte aligned", i);
    EmaSegDev e;
    e.src = g.src;
    e.dst = g.dst;
    e.mode = g.mode;
    e.vec = ((s ^ d) & 15u) == 0;
    e.head = e.vec ? (int)std::min<int64_t>(((16 - (d & 15u)) & 15u) / 4, g.n) : 0;
    e.quads = (g.n - e.head) / 4;
    e.tail = (int)(g.n - e.head - 4 * e.quads);
    e.chunk0 = chunks;
    chunks += std::max<int64_t>(1, ceil_div(e.quads, kEmaChunkQuads));
    segs.push_back(e);
  }
  if (segs.empty()) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  KDB_CUDA(cudaStreamIsCapturing(st, &cap));
  KDB_REQUIRE(cap == cudaStreamCaptureStatusNone, KDB_ERR_UNSUPPORTED,
              "ema_update: not capturable (the segment table is copied from a host buffer reused by the next call)");
  int device = 0;
  KDB_CUDA(cudaGetDevice(&device));
  std::lock_guard<std::mutex> lock(g_ema_mutex);
  EmaTable* t = nullptr;
  if (int rc = ema_table(device, segs.size(), t)) return rc;
  KDB_CUDA(cudaEventSynchronize(t->copied));   // the previous call's copy has left the staging buffer
  std::copy(segs.begin(), segs.end(), t->pinned);
  KDB_CUDA(cudaStreamWaitEvent(st, t->done, 0));   // and its kernel has finished reading the device table
  KDB_CUDA(cudaMemcpyAsync(t->dev, t->pinned, segs.size() * sizeof(EmaSegDev), cudaMemcpyHostToDevice, st));
  KDB_CUDA(cudaEventRecord(t->copied, st));
  const unsigned grid = (unsigned)std::min<int64_t>(chunks, (int64_t)kNumSMs * (2048 / kEmaThreads));
  ema_update_kernel<<<grid, kEmaThreads, 0, st>>>(t->dev, (int)segs.size(), chunks, weight);
  KDB_LAUNCH_CHECK(F_EMA, st);
  KDB_CUDA(cudaEventRecord(t->done, st));
  return 0;
}

}  // extern "C"
