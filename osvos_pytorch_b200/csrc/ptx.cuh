// Thin inline-PTX wrappers for the sm_90a features the OSVOS kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors (wgmma.cuh holds the MMA itself).
// Hand-written; encodings follow the PTX ISA chapter on warpgroup-level matrix multiply.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace osvos {

#ifndef OSVOS_SPIN_LIMIT
// Every mbarrier wait is bounded: a protocol bug must surface as a trap
// (cudaErrorLaunchFailure), never as a hung GPU.
#define OSVOS_SPIN_LIMIT (1u << 26)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------- programmatic dependent launch
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while the previous kernel
// of the stream is still draining.  pdl_wait() blocks until that kernel has COMPLETED and its memory is visible
// (a no-op for a normal launch): nothing written by an earlier kernel may be read, and nothing it reads may be
// overwritten, before this point.  pdl_launch_dependents() lets the NEXT kernel's blocks be scheduled as soon as
// every block of this grid has issued it (they then park in their own pdl_wait()).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > OSVOS_SPIN_LIMIT) __trap();
  }
}

// ----------------------------------------------------- cp.async (non-bulk) into an mbarrier-tracked stage
// 8-byte asynchronous copy global -> shared; src_bytes = 0 zero-fills the destination (out-of-image elements).
__device__ __forceinline__ void cp_async_8_zfill(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
// The executing thread's prior cp.async operations arrive on `bar` when they complete; .noinc: the arrival must be part
// of the barrier's initial count.
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// Shared -> global tensor store; elements outside the tensor's bounds are skipped.  The source must have been written
// before a fence.proxy.async (fence_proxy_async_smem) by every thread that wrote it.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// Closes the calling thread's bulk group of the stores issued since the last commit.
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Waits until at most N of the calling thread's bulk groups are pending: .read only until their shared-memory sources
// have been read (the source may then be rewritten), the plain form until their writes are complete.
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// --------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor (64 bit):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset>>4 [49,52) base offset (0: the swizzle follows the absolute address)
//   [62,64) layout: 0 none, 1 SW128, 2 SW64, 3 SW32
// Descriptors are advanced by ADDING (bytes >> 4): shared-memory addresses stay below 2^18, so the add never carries out
// of the start-address field.
constexpr uint64_t kDescSW128 = 1ull << 62;
__host__ __device__ constexpr uint64_t desc_template(uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout) {
  return (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16) | (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32) |
         layout;
}
__device__ __forceinline__ uint64_t make_smem_desc(const void* p, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout) {
  return desc_template(lbo_bytes, sbo_bytes, layout) | static_cast<uint64_t>((smem_u32(p) >> 4) & 0x3FFF);
}

// Named barrier over `nthreads` threads (a multiple of 32) of the CTA; ids 1.. (0 is __syncthreads).
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Counts the calling warp toward named barrier `id` without waiting for it; the threads that bar.sync it wait.
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Per-thread register budget of the calling warpgroup (all four warps execute it): dec hands registers back to the SM's
// pool, inc waits until it can take them.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// Stage bookkeeping of a consumer warpgroup: a shared-memory stage may be handed back to the producer only once the wgmma
// groups reading it have completed.  With one group in flight (wgmma_wait<1>) that is the PREVIOUS group's stage.
struct StageRelease {
  uint64_t* bar_b = nullptr;
  uint64_t* bar_a = nullptr;
  __device__ __forceinline__ void release(bool leader) {
    if (leader) {
      if (bar_b) mbar_arrive(bar_b);
      if (bar_a) mbar_arrive(bar_a);
    }
    bar_b = bar_a = nullptr;
  }
};

}  // namespace osvos
