// tc_common.cuh -- sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (warpgroup MMA) and its shared-memory descriptors.
// Bit layouts follow the PTX ISA "asynchronous warpgroup level matrix shared memory layout / matrix descriptor".
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "pipe_state.cuh"

namespace kdb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- programmatic dependent launch
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in the stream is
// still running; pdl_wait() blocks until the predecessor has completed and its writes are visible (KDB_PDL_TRIGGER, common.cuh,
// lets the next kernel start).  A no-op for ordinary launches.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- persistent kernels
// The kernel's dynamic shared memory from its first 1024-byte boundary on (SWIZZLE_128B tiles need that alignment); the kernels
// request 1 KiB more than their layout for it.
__device__ __forceinline__ uint8_t* smem_1k() {
  extern __shared__ uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
}
// How many of `tiles` this CTA owns: a persistent CTA takes tiles blockIdx.x, + gridDim.x, ...
__device__ __forceinline__ int tiles_owned(int tiles) {
  return (int)blockIdx.x < tiles ? (tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// One probe of the phase.  The suspend-time hint lets the hardware park the thread until the phase completes (or the hint
// expires) instead of returning after ~100 cycles: warps that wait no longer burn issue slots their scheduler's working warps
// (epilogue arithmetic, the MMA warpgroup) need.
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(200000u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug traps after 2 s instead of hanging the GPU.  No message: a kernel whose function body contains a call
// (printf is one) gets every wgmma serialised by ptxas (each one waited for before the next issues) and the caller-saved registers
// around the call spilled.
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if ((++spins & 63u) == 0 && globaltimer_ns() - t0 > 2000000000ull) __trap();
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// store: shared (SWIZZLE_128B tile) -> global, bulk-group completion
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void named_barrier_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
// arrive without waiting: the other `threads - 32 k` threads of the barrier wait on it with named_barrier_sync
__device__ __forceinline__ void named_barrier_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// Hand registers between warpgroups (every warp of the warpgroup executes it): a producer warpgroup gives up what its MMA
// warpgroups then take, within the CTA's allocation at launch (168 per thread for the 384-thread kernels: 128 x 40 + 256 x 232).
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
constexpr uint32_t PRODUCER_REGS = 40, MMA_REGS = 232;

// ---------------------------------------------------------------- warp-specialized kernels
// Named barriers; id 0 is __syncthreads.  BAR_WG + wg: the 128 threads of MMA warpgroup wg.  BAR_TURN + wg: both MMA warpgroups,
// warpgroup wg may issue its next block of MMAs.  BAR_ACC + wg: both MMA warpgroups, wg may write the GEMM's fp32 accumulator tile.
enum : int { BAR_WG = 1, BAR_TURN = 3, BAR_ACC = 5 };
// Who releases a ring slot: the arrival count of its `empty` barrier
constexpr uint32_t REL_WARPS = 4;                  // lane 0 of each warp of one warpgroup
constexpr uint32_t REL_WARPS_2WG = 2 * REL_WARPS;  // ... of both MMA warpgroups
constexpr uint32_t REL_THREAD_2WG = 2;             // one thread of each MMA warpgroup

// N buffers filled by TMA from one producer thread.  full[s] completes when slot s has landed, empty[s] when it is released.
template <int N>
struct TmaRing {
  uint64_t full[N], empty[N];
  __device__ __forceinline__ void init(uint32_t releasers) {   // by one thread, before fence_barrier_init
    for (int s = 0; s < N; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], releasers);
    }
  }
  // producer: wait for the slot's releases, arm `full` for `bytes` and return it for the slot's TMA loads
  __device__ __forceinline__ uint64_t* acquire(PipeState<N> ps, uint32_t bytes) {
    mbar_wait_nocall(&empty[ps.slot], ps.producer_parity());
    mbar_arrive_expect_tx(&full[ps.slot], bytes);
    return &full[ps.slot];
  }
  __device__ __forceinline__ void wait(PipeState<N> ps) { mbar_wait_nocall(&full[ps.slot], ps.consumer_parity()); }
  __device__ __forceinline__ void release(PipeState<N> ps) { mbar_arrive(&empty[ps.slot]); }
};

// byte offset of 16-byte chunk `chunk16` (0..7) of `row` inside a [rows x 128 B] SWIZZLE_128B tile (what TMA / UMMA expect)
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk16) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk16 ^ (row & 7)) << 4));
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// Issued by all 128 threads of a warpgroup; the fp32 accumulator lives in their registers.  Fragment of m64nNk16: thread t of
// the warpgroup holds, for every 8-column block j, d[4j], d[4j+1] = (row 16 (t / 32) + (t % 32) / 4, columns 8j + 2 (t % 4) + {0, 1})
// and d[4j+2], d[4j+3] = the same columns of row + 8.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// ties the accumulator registers to a point in the instruction stream (no read or write of them is moved across it)
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void wg_fence_acc(uint32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// D[64 x 128] (+)= A[smem, K-major] * B[smem, K-major]^T, bf16 in, fp32 accumulate
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 64] (+)= A[smem, K-major] * B[smem]; TB = 1: B is MN-major (N contiguous), as a V tile of attention is
template <int TB>
__device__ __forceinline__ void wgmma_64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TB));
}
// D[64 x 128] (+)= A[registers: m64k16 bf16 fragment, 4 x bf16x2] * B[smem, K-major]^T
__device__ __forceinline__ void wgmma_128_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// the same with fp16 operands: A a m64k16 fp16 fragment (4 x f16x2, the lower k index in the low half), B fp16 K-major
__device__ __forceinline__ void wgmma_128_rs_f16(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// D[64 x 64] (+)= A[registers: m64k16 bf16 fragment] * B[smem]; TB = 1: B is MN-major (N contiguous)
template <int TB>
__device__ __forceinline__ void wgmma_64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate), "n"(TB));
}

// D[64 x 128] (+)= A[smem, K-major] * B[smem, K-major]^T, tf32 in (the low 13 mantissa bits of each fp32 operand are ignored), fp32
// accumulate.  A k8 step is 32 B along K, the same descriptor advance as a bf16 k16 step.
__device__ __forceinline__ void wgmma_128_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Accumulator fragment of rows [row0, row0 + 64) -> fp32 shared-memory tile, row-major with `ld` floats per row: the row-per-thread
// epilogues then read whole rows (acc_ld32).
template <int R>
__device__ __forceinline__ void acc_store(float* s, int ld, int row0, const float (&d)[R]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(s + (size_t)r * ld + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(s + (size_t)(r + 8) * ld + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// 32 consecutive fp32 columns of one row of such a tile
__device__ __forceinline__ void acc_ld32(const float* s, int ld, int row, int col0, float (&v)[32]) {
  const float4* src = reinterpret_cast<const float4*>(s + (size_t)row * ld + col0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 q = src[i];
    v[4 * i] = q.x;
    v[4 * i + 1] = q.y;
    v[4 * i + 2] = q.z;
    v[4 * i + 3] = q.w;
  }
}

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// fused RMSNorm: sum of the first `parts` (1..8) per-128-channel slots of one row-statistics record.  Exactly `parts` slots are
// read: the producers write only C / 128 of the 8 slots, the rest of the record is uninitialised workspace.
__device__ __forceinline__ float rowss_sum(const float4 s0, const float4 s1, const int parts) {
  const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  float acc = sv[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) acc += i < parts ? sv[i] : 0.f;
  return acc;
}

// ---------------------------------------------------------------- fp32 pairs
// The epilogues work on neighbouring columns in pairs; every operation is the scalar .rn one.
struct f32x2 {
  float x, y;
};
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
  lo = v.x;
  hi = v.y;
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return f32x2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f32x2 neg2(f32x2 a) { return f32x2{-a.x, -a.y}; }
// (2 * half_val) * gelu_tanh(gate) for two (value, gate) pairs, GELU in the tanh form on the MUFU tanh unit: |gelu_tanh - gelu_erf|
// <= 5e-4 absolute, below one bf16 ulp wherever the output magnitude exceeds 0.07 -- used only on the bf16 fast path; the fp32
// path keeps erff.  `half_val` = 0.5 * value (the caller folds the 0.5 into the row scale it applies anyway):  val * gate * (0.5 + 0.5 t) = w + w t  with w = half_val * gate  -> 5 packed instructions + 2 MUFU
__device__ __forceinline__ f32x2 geglu2(f32x2 half_val, f32x2 gate) {
  const f32x2 c1 = pk2(0.0356774081f, 0.0356774081f), c0 = pk2(0.7978845608f, 0.7978845608f);
  const f32x2 u = mul2(gate, fma2(c1, mul2(gate, gate), c0));
  float u0, u1;
  upk2(u, u0, u1);
  const f32x2 t = pk2(tanh_approx(u0), tanh_approx(u1));
  const f32x2 w = mul2(half_val, gate);
  return fma2(w, t, w);
}

// ---------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor, 128B swizzle: bits [0,14) start >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [62,64) layout = 1 (SW128).
// K-major operand tile whose rows are 128 bytes (64 bf16) wide, 8-row groups 1024 B apart (LBO unused).  A K step of 16 bf16 = 32 B
// inside the swizzle atom is +2 on the descriptor.
__device__ __forceinline__ uint64_t smem_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// 64B swizzle: K-major tile whose rows are 64 bytes (32 fp16) wide, 8-row groups 512 B apart; a K step of 16 fp16 = 32 B is +2.
__device__ __forceinline__ uint64_t smem_desc_k_sw64(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (32ull << 32) | (2ull << 62);
}
// MN-major operand tile (rows of the *K* index are 128 B = 64 bf16 of the MN index): 64-element MN atoms LBO apart, 8-row K groups SBO apart.
__device__ __forceinline__ uint64_t smem_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void unpack_bf16x2(uint32_t v, float& lo, float& hi) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&v);
  lo = __low2float(t);
  hi = __high2float(t);
}

// GEGLU on a wgmma accumulator fragment of 64 rows x 128 columns whose W rows interleave 8 value / 8 gate rows: 8-column block 2q holds
// 8 value features, block 2q + 1 their gates, so a value and its gate sit in the same thread.  h0 / h1: 0.5 x the value scale of the
// thread's rows r, r + 8 (the GELU's 0.5 rides on it); g0 / g1: their gate scale.  o[2q] / o[2q + 1]: hidden features 8q + cq, 8q + cq + 1
// of row r / r + 8 as bf16x2 -- which is also the bf16 A fragment of k16 step q / 2 (wgmma_128_rs).
__device__ __forceinline__ void geglu_fragment(const float (&acc)[64], f32x2 h0, f32x2 h1, f32x2 g0, f32x2 g1, uint32_t (&o)[16]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const f32x2 v0 = mul2(pk2(acc[8 * q], acc[8 * q + 1]), h0), v1 = mul2(pk2(acc[8 * q + 2], acc[8 * q + 3]), h1);
    const f32x2 q0 = mul2(pk2(acc[8 * q + 4], acc[8 * q + 5]), g0), q1 = mul2(pk2(acc[8 * q + 6], acc[8 * q + 7]), g1);
    float o0, o1, o2, o3;
    upk2(geglu2(v0, q0), o0, o1);
    upk2(geglu2(v1, q1), o2, o3);
    o[2 * q] = pack_bf16x2(o0, o1);
    o[2 * q + 1] = pack_bf16x2(o2, o3);
  }
}

// ---------------------------------------------------------------- shifted windows of 8x8 tokens (reference image_transformer_v2.py:253-337)
// A window moves as four 4x4-token quadrant boxes; its rows are quadrant-major, then (row, column) inside the quadrant.
// window `win` of a [B, h, w] token grid -> image b, window row wi, window column wj
__device__ __forceinline__ void window_coords(int win, int h, int w, int& b, int& wi, int& wj) {
  const int nww = w >> 3, per_img = (h >> 3) * nww;
  b = win / per_img;
  const int rem = win - b * per_img;
  wi = rem / nww;
  wj = rem - wi * nww;
}
// origin of quadrant q of window (wi, wj) in original coordinates: the roll of the shifted layers (:274)
__device__ __forceinline__ void quad_origin(int wi, int wj, int q, int h, int w, int shift, int& r, int& c) {
  r = (wi * 8 + (q >> 1) * 4 - shift + h) % h;
  c = (wj * 8 + (q & 1) * 4 - shift + w) % w;
}
// seam mask (:300-315): in the top (seam_r) / left (seam_c) windows of a shifted layer a query of quadrant qq sees a key of quadrant kq
// only on its own side of the wrapped row / column
__device__ __forceinline__ bool seam_ok(int qq, int kq, bool seam_r, bool seam_c) {
  return (!seam_r || ((kq >> 1) == (qq >> 1))) && (!seam_c || ((kq & 1) == (qq & 1)));
}

// ---------------------------------------------------------------- attention on a register score fragment
// One key block of O = softmax(S) V for the 64 query rows of a warpgroup.  s: S [64 x NK] as a wgmma fragment (rows rw, rw + 8, column
// pair 2 (t % 4) of every 8-column block c); key_ok(c): block c's keys are visible.  mx0 / mx1: the rows' maxima so far (BOUNDED: the
// fixed shift exp(s - bound)); l0 / l1: this thread's part of the rows' sums of P; o += P V.  Without the bound, when `rescale` (a later
// key block) l and o are rescaled from the old maximum to the new one.  P is rounded to bf16, the register A operand of the P V wgmma,
// and l sums the rounded values.  vdesc: V [NK keys x 64] bf16, an MN-major SW128 operand.
template <int NK, bool BOUNDED, typename KeyOk>
__device__ __forceinline__ void softmax_pv(float (&s)[NK / 2], const KeyOk& key_ok, bool rescale, float& mx0, float& mx1, float& l0, float& l1,
                                           float (&o)[32], uint64_t vdesc) {
  constexpr float LOG2E = 1.4426950408889634f;
  if constexpr (!BOUNDED) {
    float n0 = mx0, n1 = mx1;
#pragma unroll
    for (int c = 0; c < NK / 8; ++c) {
      if (!key_ok(c)) s[4 * c] = s[4 * c + 1] = s[4 * c + 2] = s[4 * c + 3] = -INFINITY;
      n0 = fmaxf(n0, fmaxf(s[4 * c], s[4 * c + 1]));
      n1 = fmaxf(n1, fmaxf(s[4 * c + 2], s[4 * c + 3]));
    }
    n0 = fmaxf(n0, __shfl_xor_sync(0xffffffffu, n0, 1));
    n0 = fmaxf(n0, __shfl_xor_sync(0xffffffffu, n0, 2));
    n1 = fmaxf(n1, __shfl_xor_sync(0xffffffffu, n1, 1));
    n1 = fmaxf(n1, __shfl_xor_sync(0xffffffffu, n1, 2));
    if (rescale) {                             // the maximum grew: rescale what was accumulated against the old one
      const float a0 = exp2f((mx0 - n0) * LOG2E), a1 = exp2f((mx1 - n1) * LOG2E);
      l0 *= a0;
      l1 *= a1;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        o[4 * c] *= a0;
        o[4 * c + 1] *= a0;
        o[4 * c + 2] *= a1;
        o[4 * c + 3] *= a1;
      }
    }
    mx0 = n0;
    mx1 = n1;
  }
  const float mb0 = mx0 * LOG2E, mb1 = mx1 * LOG2E;
  uint32_t pf[NK / 4];
#pragma unroll
  for (int i2 = 0; i2 < NK / 4; ++i2) {
    const float mb = (i2 & 1) ? mb1 : mb0;
    float p0 = exp2f(fmaf(s[2 * i2], LOG2E, -mb)), p1 = exp2f(fmaf(s[2 * i2 + 1], LOG2E, -mb));
    if (BOUNDED && !key_ok(i2 >> 1)) p0 = p1 = 0.f;   // (bounded) zero probability instead of a -inf logit
    pf[i2] = pack_bf16x2(p0, p1);
    float e0, e1;
    unpack_bf16x2(pf[i2], e0, e1);             // l accumulates exactly what the P V MMA sees
    if (i2 & 1) l1 += e0 + e1;
    else l0 += e0 + e1;
  }
  // ---- O += P V, 16 keys per step: rows 16 kk.. of V
  wg_fence_acc(o);
  wg_fence_acc(pf);
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < NK / 16; ++kk) {
    const uint32_t a[4] = {pf[4 * kk], pf[4 * kk + 1], pf[4 * kk + 2], pf[4 * kk + 3]};
    wgmma_64_rs<1>(o, a, vdesc + (uint64_t)(kk * ((16 * 128) >> 4)), 1u);
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(o);
}
// after the last key block: O / l, l summed over the quad that holds a row
__device__ __forceinline__ void softmax_normalize(float (&o)[32], float l0, float l1) {
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = __frcp_rn(l0), inv1 = __frcp_rn(l1);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    o[4 * c] *= inv0;
    o[4 * c + 1] *= inv0;
    o[4 * c + 2] *= inv1;
    o[4 * c + 3] *= inv1;
  }
}

// ---------------------------------------------------------------- residual epilogue of the fused kernels
// x += acc in place, where acc is a thread's fragment of 64 rows x 128 columns (rows r, r + 8, column pair cq of every 8-column block)
// and x a bf16 tile of 128 columns held as two [128 x 64] SW128 halves of 16 KiB.  Returns the two rows' sums of squares of the new x,
// reduced over the quad.
__device__ __forceinline__ float2 residual_add(uint8_t* xt, int r, int cq, const float (&acc)[64]) {
  float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    uint8_t* sub = xt + (j >> 3) * (128 * 128);
    uint32_t* p0 = reinterpret_cast<uint32_t*>(sub + sw128_offset(r, j & 7) + cq * 2);
    uint32_t* p1 = reinterpret_cast<uint32_t*>(sub + sw128_offset(r + 8, j & 7) + cq * 2);
    const uint32_t x0 = *p0, x1 = *p1;
    const float a0 = acc[4 * j] + __uint_as_float(x0 << 16), a1 = acc[4 * j + 1] + __uint_as_float(x0 & 0xffff0000u);
    const float b0 = acc[4 * j + 2] + __uint_as_float(x1 << 16), b1 = acc[4 * j + 3] + __uint_as_float(x1 & 0xffff0000u);
    ss0 = fmaf(a0, a0, fmaf(a1, a1, ss0));
    ss1 = fmaf(b0, b0, fmaf(b1, b1, ss1));
    *p0 = pack_bf16x2(a0, a1);
    *p1 = pack_bf16x2(b0, b1);
  }
  ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1);
  ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
  ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1);
  ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
  return make_float2(ss0, ss1);
}

}  // namespace tc

// ---------------------------------------------------------------- host: tensor maps
// 2-D..4-D bf16 tensor map with 128B swizzle; dims/strides innermost first (strides in bytes, for dims 1..rank-1).
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
// the same for fp32 elements (a 128-byte swizzle row is 32 of them); out-of-bounds box elements read as zeros
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);
// fp16 elements with a 64-byte swizzle (a 32-element row is one 64-byte swizzle row); out-of-bounds box elements read as zeros
int make_tmap_f16_sw64(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                       const uint32_t* box);
// [B, h, w, C] bf16 tokens as the 4-D map (C, w, h, B) with box {box_c, box_w, box_h, 1}
int make_tmap_tokens(CUtensorMap* out, const void* base, uint64_t C, int B, int h, int w, uint32_t box_c, uint32_t box_w, uint32_t box_h);

// SM count of the current device: the grid of the persistent kernels
inline int num_sms() {
  static int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = kNumSMs;
    return v;
  }();
  return n;
}
// grid of a persistent kernel over `tiles` tiles: min(tiles, SMs) CTAs
inline dim3 persistent_grid(int64_t tiles) { return dim3((unsigned)(tiles < num_sms() ? tiles : num_sms())); }

// ---------------------------------------------------------------- host: programmatic dependent launch
// Launches `kernel` with programmatic stream serialization, so that its prologue overlaps the tail of the previous kernel in the
// stream (the kernel calls pdl_wait() before it reads that kernel's output).  In plain stream order when pdl_enabled() is false.
bool pdl_enabled();
template <typename... Params, typename... Args>
cudaError_t launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t lc{};
  lc.gridDim = grid;
  lc.blockDim = block;
  lc.dynamicSmemBytes = smem;
  lc.stream = st;
  lc.attrs = attr;
  lc.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&lc, kernel, args...);
}

}  // namespace kdb
