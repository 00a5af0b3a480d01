// mbarrier / TMA bulk-copy primitives shared by the kernels (inline PTX, sm_90+; SASS: SYNCS.*, UBLKCP)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace eb {

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait.  The bound is a last-resort guard against hanging the GPU on a lost partner (a trap is
// an error the host reports); it must exceed every legitimate wait, including a producer that is itself
// waiting for a peer GPU (30 s bound there), hence ~2 minutes.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 240000000000ll) __trap();
  }
}
// Abortable wait for kernels whose producers may give up on a lost peer GPU: `abort` is a CTA-wide
// shared-memory flag the producers set on a barrier timeout; every warp of the CTA then leaves
// instead of spinning into the trap, and the host reports FLAG_COMM_TIMEOUT as EB_ERR_COMM.
__device__ __forceinline__ bool mbar_wait_abortable(uint64_t* bar, unsigned parity, const volatile int* abort) {
  if (mbar_try_wait(bar, parity)) return true;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (*abort) return false;
    if (clock64() - t0 > 240000000000ll) __trap();
  }
  return true;
}
// The same wait without the trap, for code that runs under a limit raised by setmaxnreg.inc: ptxas (CUDA 12.9)
// does not give code from which a trap is reachable the raised limit.  At the last-resort bound it ORs
// `timeout_flag` into the status word and raises `abort` itself, so the other warps leave as well.
__device__ __forceinline__ bool mbar_wait_abortable_notrap(uint64_t* bar, unsigned parity, volatile int* abort,
                                                           int* status, int timeout_flag) {
  if (mbar_try_wait(bar, parity)) return true;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (*abort) return false;
    if (clock64() - t0 > 240000000000ll) {
      atomicOr(status, timeout_flag);
      *abort = 1;
      return false;
    }
  }
  return true;
}
// best-effort wait of at most `cycles`: for orderings that are optimisations, not dependencies
__device__ __forceinline__ void mbar_wait_for(uint64_t* bar, unsigned parity, long long cycles) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > cycles) return;
  }
}
// global -> shared bulk copy (TMA, SASS UBLKCP); completion is counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// the same copy with an L2 eviction priority (`policy` from l2_evict_first_policy)
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, unsigned bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// L2 cache policy: the lines a copy brings in are the first to be evicted
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// shared -> global bulk copy (TMA store); completion tracked by the thread's bulk async-group
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread have finished READING shared memory
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory -> visible to the async proxy (TMA store source)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }


// programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization
// attribute starts while its predecessor in the stream is still draining; everything that reads or
// writes what the predecessor touches sits behind pdl_wait().  Both are no-ops for a plain launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// pull one 128-byte line into L2 (no register, no L1 allocation)
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

}  // namespace eb
