// tc_common.cuh -- sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (warpgroup MMA) and its shared-memory descriptors.
// Bit layouts follow the PTX ISA "asynchronous warpgroup level matrix shared memory layout / matrix descriptor".
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace kdb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- programmatic dependent launch
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in the stream is
// still running; pdl_wait() blocks until the predecessor has completed and its writes are visible.  pdl_launch_dependents()
// tells the scheduler that the NEXT kernel's CTAs may be placed as soon as this grid's CTAs have all passed this point (or
// exited) and resources free up.  Both are no-ops for ordinary launches.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

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
// Bounded wait: a protocol bug traps after 2 s with a message instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 63u) == 0 && globaltimer_ns() - t0 > 2000000000ull) {
      printf("libkdb200: mbarrier wait timed out (block %d,%d,%d thread %d parity %u)\n", blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x, parity);
      __trap();
    }
  }
}

// Wait of a SINGLE-THREAD role (TMA producer, MMA issuer): the parked wait above goes to sleep (NANOSLEEP.SYNCS) when the phase is not
// complete yet and pays the wake-up on the hand-off's critical path; a lone thread that polls costs no other warp an issue slot worth
// having.  KDB_SPIN_ROLES: 0 = parked waits everywhere (default), 1 = the single-thread roles poll, 2 = also the epilogue groups'
// accumulator waits.
// Bounded like mbar_wait.
#ifndef KDB_SPIN_ROLES
#define KDB_SPIN_ROLES 0
#endif
__device__ __forceinline__ bool mbar_try_wait_nohint(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait_nohint(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait_nohint(bar, parity)) {
    if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > 2000000000ull) {
      printf("libkdb200: mbarrier wait timed out (block %d,%d,%d thread %d parity %u)\n", blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x, parity);
      __trap();
    }
  }
}
__device__ __forceinline__ void mbar_wait_role(uint64_t* bar, uint32_t parity) {
  if (KDB_SPIN_ROLES >= 1) mbar_wait_spin(bar, parity);
  else mbar_wait(bar, parity);
}
__device__ __forceinline__ void mbar_wait_group(uint64_t* bar, uint32_t parity) {
  if (KDB_SPIN_ROLES >= 2) mbar_wait_spin(bar, parity);
  else mbar_wait(bar, parity);
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
// store: shared (SWIZZLE_128B tile) -> global, bulk-group completion
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read_le1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void named_barrier_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

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

// 2^x on the MUFU unit, flush-to-zero: for softmax terms (x <= ~0; results below 2^-126 are irrelevant)
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// GELU in the tanh form on the MUFU tanh unit (6 instructions).  |gelu_tanh - gelu_erf| <= 5e-4 absolute, i.e. below one
// bf16 ulp wherever the output magnitude exceeds 0.07 -- used only on the bf16 fast path; the fp32 path keeps erff.
__device__ __forceinline__ float gelu_fast(float x) {
  const float u = x * fmaf(0.0356774081f, x * x, 0.7978845608f);     // sqrt(2/pi) (x + 0.044715 x^3)
  return x * fmaf(0.5f, tanh_approx(u), 0.5f);
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
// (2 * half_val) * gelu_fast(gate) for two (value, gate) pairs; `half_val` = 0.5 * value (the caller folds the 0.5 into the
// row scale it applies anyway):  val * gate * (0.5 + 0.5 t) = w + w t  with w = half_val * gate  -> 5 packed instructions + 2 MUFU
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

}  // namespace tc

// ---------------------------------------------------------------- host: tensor maps
// 2-D..4-D bf16 tensor map with 128B swizzle; dims/strides innermost first (strides in bytes, for dims 1..rank-1).
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);

}  // namespace kdb
