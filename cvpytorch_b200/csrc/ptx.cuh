// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma shared-memory matrix descriptors.
// Written for this project; bit layouts follow the PTX ISA tables for wgmma matrix descriptors.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace cvb {

#ifndef CVB_WATCHDOG
#define CVB_WATCHDOG 1  // trap instead of hanging forever if a pipeline barrier never flips
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\telect.sync R|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// same with a suspend-time hint (ns): the thread may sleep in hardware up to that long before the instruction returns false
__device__ __forceinline__ uint32_t mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t hint) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(hint)
      : "memory");
  return ok;
}
// `tag` identifies the waiter in the watchdog message (printed only when built with -DCVB_WATCHDOG=2: the printf call site costs
// ~30 instructions and a stack frame per inlined wait, and the single-thread producer / MMA loops are instruction-latency bound).
// `hint` > 0: long waits (a producer waiting for a free ring slot) sleep in hardware instead of spinning on the issue port.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag, uint32_t hint = 0) {
#if CVB_WATCHDOG
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!(hint ? mbar_try_wait_hint(bar, parity, hint) : mbar_try_wait(bar, parity))) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz: trap instead of hanging the GPU
#if CVB_WATCHDOG >= 2
      printf("[cvb200] mbarrier watchdog: block %d thread %d tag %d parity %u\n", (int)blockIdx.x, (int)threadIdx.x, tag, parity);
#endif
      __trap();
    }
  }
#else
  while (!(hint ? mbar_try_wait_hint(bar, parity, hint) : mbar_try_wait(bar, parity))) {
  }
#endif
  (void)tag;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
// 1D bulk copy shared -> global (both 16-byte aligned, size a multiple of 16), tracked by the issuing thread's bulk groups
__device__ __forceinline__ void bulk_store_1d(void* gdst, const void* smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(reinterpret_cast<uint64_t>(gdst)), "r"(smem_u32(smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- programmatic dependent launch
// wait: blocks until every prerequisite grid has completed and its memory is visible (no-op without the launch attribute).
// launch_dependents: lets the next kernel in the stream start its prologue once all CTAs of this grid have passed this point.
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// K-major shared-memory operand descriptor (wgmma "matrix descriptor"), swizzled layouts.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1)
//   bits [32,46) stride byte offset >> 4   (distance between 8-row groups = 8 * swizzle bytes)
//   bits [62,64) layout: 1 = 128B swizzle, 2 = 64B, 3 = 32B  (written below as the 3-bit field at 61: 2, 4, 6)
template <int SWIZZLE_BYTES>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
  constexpr uint64_t layout = SWIZZLE_BYTES == 128 ? 2ull : (SWIZZLE_BYTES == 64 ? 4ull : 6ull);
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8u * SWIZZLE_BYTES) >> 4) << 32;
  d |= layout << 61;
  return d;
}
// Same, with an explicit stride byte offset (pitch between 8-row groups).  Used by the halo-tile 3x3 path: the rows of a
// tap-shifted A tile are pixels of one halo image, 8 consecutive pixels per group, groups one image row (16 pixels) apart.
// The hardware applies the swizzle XOR on absolute shared-memory address bits, so a start address shifted by whole rows
// stays consistent with what TMA wrote.
template <int SWIZZLE_BYTES>
__device__ __forceinline__ uint64_t make_kmajor_desc_sbo(uint32_t smem_addr, uint32_t sbo_bytes) {
  constexpr uint64_t layout = SWIZZLE_BYTES == 128 ? 2ull : (SWIZZLE_BYTES == 64 ? 4ull : 6ull);
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(sbo_bytes >> 4) << 32;
  d |= layout << 61;
  return d;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

}  // namespace cvb
