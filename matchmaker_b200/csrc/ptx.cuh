// Thin inline-PTX wrappers for the sm_90a features the interaction kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors), proxies,
// clusters.  Hand-written for this project; bit layouts follow the PTX ISA descriptions of the wgmma
// shared-memory matrix descriptor and of the wgmma accumulator fragments.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mmb {

// ---------------------------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }


// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(
                   smem_u32(bar)),
               "r"(bytes)
               : "memory");
}

// Blocking wait: try_wait returns at once when the phase is still open; the loop re-issues it and checks a clock
// watchdog, so a protocol bug ends in a trap (the launch fails with an error the host reports) instead of a hung GPU.
// No printf in the product build: any function call in a kernel makes ptxas serialise its wgmma pipeline (and spill
// around the call).  Debugging builds (-DMMB200_ENABLE_PROF) print which barrier timed out.
//
// Parity waits are unambiguous only while the barrier is at most one phase behind the phase waited for: every barrier
// here has waiters that pass through all of its phases in order.
#ifndef MMB_WATCHDOG_CYCLES
#define MMB_WATCHDOG_CYCLES (4000000000ll)  // ~2 s at 1.98 GHz
#endif

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
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

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > MMB_WATCHDOG_CYCLES) {
#ifdef MMB200_ENABLE_PROF
      printf("mmb200: mbarrier watchdog (block %d thread %d bar %u parity %u)\n", (int)blockIdx.x, (int)threadIdx.x,
             smem_u32(bar), parity);
#endif
      __trap();
    }
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, void* smem_dst, uint64_t* bar, int c0,
                                            int c1, int c2, int c3, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "l"(cache_hint)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, void* smem_dst, uint64_t* bar, int c0,
                                            int c1, int c2, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(cache_hint)
      : "memory");
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, void* smem_dst, uint64_t* bar, int c0,
                                            int c1, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(cache_hint)
      : "memory");
}

// 16-byte cp.async (L2 only) of which the first `src_bytes` (16 or 0) are read; the rest of the 16 bytes is zero-filled.
__device__ __forceinline__ void cp_async_16_zfill(uint32_t smem_dst, const void* gmem_src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(gmem_src)),
               "r"(src_bytes)
               : "memory");
}

// One arrival on `bar` once every cp.async this thread issued so far has landed.  .noinc: the arrival counts against
// the barrier's expected count, which has to include it.
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Plain bulk copy (no tensor map): `bytes` (a multiple of 16) from 16-byte aligned global memory to 16-byte aligned shared
// memory; completion is signalled as transaction bytes on `bar`.
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[64 x N] (+)= A[64 x K] * B[N x K]^T, issued by all 128 threads of a warpgroup (4 consecutive
// warps starting at a multiple of 4), accumulator in registers.  Fragment of thread (warp w of the warpgroup, lane l),
// for every 8-column group j:  d[4j + 0..1] = row 16w + l/4,     columns 8j + 2(l%4) + 0..1
//                              d[4j + 2..3] = row 16w + l/4 + 8, same columns
// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor for a K-major operand stored as rows of exactly 128 bytes (64 x 16-bit or 32 x 32-bit
// elements along K) written by TMA with CU_TENSOR_MAP_SWIZZLE_128B:
//   bits [0,14)  start address >> 4
//   bits [16,30) leading-dimension byte offset >> 4 (unused for swizzled K-major; canonical value 1)
//   bits [32,46) stride-dimension byte offset >> 4 = 1024 B: distance between 8-row groups
//   bits [49,52) base offset = 0 (tiles are 1024-B aligned)
//   bits [62,64) layout type: 1 = SWIZZLE_128B
// A K-step inside the 128-byte row advances the start address (32 bytes per k16 of 16-bit data).
__device__ __forceinline__ uint64_t make_wgmma_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Orders this thread's earlier register / shared-memory accesses before the wgmma that follow (all 128 threads).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most kPending committed groups of this warpgroup still in flight afterwards
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// Keeps the compiler from moving reads of an accumulator above the wgmma_wait that completes it.
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// The wrappers: accumulator operands first ("+f", NR registers), then the A descriptor / A registers, the B descriptor
// and the scale-d flag (0: D = A * B, else D += A * B), which selects the predicate p.
#define MMB_ACC4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define MMB_ACC16(i) MMB_ACC4(i), MMB_ACC4(i + 4), MMB_ACC4(i + 8), MMB_ACC4(i + 12)
#define MMB_REGS16 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define MMB_REGS20 MMB_REGS16 ", %16, %17, %18, %19"
#define MMB_REGS32 MMB_REGS16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define MMB_REGS64                                                                                               \
  MMB_REGS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                    \
             "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"

// Both operands from shared-memory descriptors (K-major).  16-bit inputs take K = 16 and the two transpose flags
// (TNSP ", 0, 0"); e4m3 inputs take K = 32 and no transpose flags (8-bit wgmma reads K-major operands only), so a k32
// e4m3 step advances the same 32 bytes along a 128-byte swizzled row as a k16 step of 16-bit data.
#define MMB_WGMMA_SS(N, K, TY, TNSP, NR, REGS, PI, AI, BI, ...)                                                      \
  __device__ __forceinline__ void wgmma_m64n##N##k##K##_##TY(float (&d)[NR], uint64_t adesc, uint64_t bdesc,           \
                                                             uint32_t accumulate) {                                  \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " PI ", 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k" #K ".f32." #TY "." #TY " {" REGS "}, " AI ", " BI          \
                 ", p, 1, 1" TNSP ";\n\t}"                                                                             \
                 : __VA_ARGS__                                                                                       \
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));                                                        \
  }
MMB_WGMMA_SS(32, 16, f16, ", 0, 0", 16, MMB_REGS16, "%18", "%16", "%17", MMB_ACC16(0))
MMB_WGMMA_SS(32, 16, bf16, ", 0, 0", 16, MMB_REGS16, "%18", "%16", "%17", MMB_ACC16(0))
MMB_WGMMA_SS(64, 16, f16, ", 0, 0", 32, MMB_REGS32, "%34", "%32", "%33", MMB_ACC16(0), MMB_ACC16(16))
MMB_WGMMA_SS(64, 16, bf16, ", 0, 0", 32, MMB_REGS32, "%34", "%32", "%33", MMB_ACC16(0), MMB_ACC16(16))
MMB_WGMMA_SS(128, 16, f16, ", 0, 0", 64, MMB_REGS64, "%66", "%64", "%65", MMB_ACC16(0), MMB_ACC16(16), MMB_ACC16(32), MMB_ACC16(48))
MMB_WGMMA_SS(128, 16, bf16, ", 0, 0", 64, MMB_REGS64, "%66", "%64", "%65", MMB_ACC16(0), MMB_ACC16(16), MMB_ACC16(32), MMB_ACC16(48))
MMB_WGMMA_SS(32, 32, e4m3, "", 16, MMB_REGS16, "%18", "%16", "%17", MMB_ACC16(0))
MMB_WGMMA_SS(128, 32, e4m3, "", 64, MMB_REGS64, "%66", "%64", "%65", MMB_ACC16(0), MMB_ACC16(16), MMB_ACC16(32), MMB_ACC16(48))

// tf32 with the A operand in registers (K = 8): thread (warp w, lane l) supplies
//   a[0] = A[16w + l/4][l%4], a[1] = A[16w + l/4 + 8][l%4], a[2] = A[16w + l/4][l%4 + 4], a[3] = A[16w + l/4 + 8][l%4 + 4]
// as tf32 bit patterns; B from a K-major SWIZZLE_128B descriptor (+32 bytes per K-step).
#define MMB_WGMMA_RS_TF32(N, NR, REGS, A0, PI, BI, ...)                                                             \
  __device__ __forceinline__ void wgmma_m64n##N##k8_tf32_rs(float (&d)[NR], const uint32_t (&a)[4], uint64_t bdesc,     \
                                                            uint32_t accumulate) {                                   \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " PI ", 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 {" REGS "}, {" A0 "}, " BI ", p, 1, 1;\n\t}"   \
                 : __VA_ARGS__                                                                                       \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));                        \
  }
MMB_WGMMA_RS_TF32(64, 32, MMB_REGS32, "%32, %33, %34, %35", "%37", "%36", MMB_ACC16(0), MMB_ACC16(16))
MMB_WGMMA_RS_TF32(40, 20, MMB_REGS20, "%20, %21, %22, %23", "%25", "%24", MMB_ACC16(0), MMB_ACC4(16))
MMB_WGMMA_RS_TF32(32, 16, MMB_REGS16, "%16, %17, %18, %19", "%21", "%20", MMB_ACC16(0))

// fp32 -> tf32, round to nearest (the tensor core itself drops the low 13 bits)
__device__ __forceinline__ uint32_t f32_to_tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// Re-deal the CTA's registers between warpgroups (4 consecutive warps, all of which must execute the instruction):
// light roles shrink, the register-hungry role grows.  The sum over the CTA must fit the registers the CTA was
// launched with.
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// ---------------------------------------------------------------------------------------------
// thread-block clusters: rank, cluster-wide barrier, TMA multicast, multicast commit
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// all threads of all CTAs of the cluster (release / acquire: mbarrier inits are visible after it)
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// one tensor-map box -> the SAME shared-memory offset of every CTA in `cta_mask`; each destination CTA's mbarrier (same
// offset) receives the complete_tx for the bytes written into it
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* map, void* smem_dst, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask), "l"(cache_hint)
      : "memory");
}
// Arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (release at cluster scope).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
// One lane of a CONVERGED warp.  TMA instructions take their operands from uniform registers: issue them
// as `if (elect_one_sync()) { ... }` from warp-uniform control flow with operands computed OUTSIDE the branch, so the
// compiler keeps them uniform.  Inside an `if (lane == 0)` region it cannot prove uniformity and wraps every
// instruction in an ELECT / R2UR.BROADCAST / BRA.U.ANY waterfall loop.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// named barriers (sub-CTA sync), ids 1..15 (0 = __syncthreads)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Arrives without waiting: the shared-memory writes before it are visible to the threads that bar.sync on the same
// barrier (nthreads counts both sides).
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// streaming global loads
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

}  // namespace mmb
