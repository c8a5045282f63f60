// tma_utils.cuh -- inline-PTX wrappers for mbarrier and TMA (cp.async.bulk.tensor) used by the sm_90a kernels.
#pragma once
#include <cuda.h>
#include <cstdint>

namespace amtk {

// ---------------------------------------------------------------------------------------------------------
// PTX helpers (mbarrier + TMA)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// the same wait for a warp that has nothing else to do: backs off between polls so that it does not take issue slots
// from the warps sharing its scheduler
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  for (;;) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (done) break;
    __nanosleep(64);
  }
}
// Watchdog wait of the ring kernels (comb_mma.cuh, the band form of comb_stream.cuh).  No wait may spin forever: after
// ~1 s a thread records (code, step, CTA, thread) in dbg[] and raises dbg[0]; from then on every wait of every CTA returns
// at once, the launch drains with garbage results and the host reports the failure.
constexpr long long kMmWaitLimit = 2000000000ll;           // clock64 ticks (~1 s)
__device__ __noinline__ void mm_wait_slow(uint64_t* bar, uint32_t parity, int* dbg, int code, int step, bool sleepy) {
  const long long t0 = clock64();
  for (uint32_t spin = 0;; ++spin) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (done) return;
    if (sleepy) __nanosleep(64);
    if ((spin & 15u) == 15u) {
      if (*reinterpret_cast<volatile int*>(dbg)) return;
      if (clock64() - t0 > kMmWaitLimit) {
        if (atomicCAS(dbg, 0, 1) == 0) { dbg[1] = code; dbg[2] = step; dbg[3] = (int)blockIdx.x; dbg[4] = (int)threadIdx.x; dbg[5] = (int)parity; __threadfence(); }
        return;
      }
    }
  }
}
__device__ __forceinline__ void mm_wait(uint64_t* bar, uint32_t parity, int* dbg, int code, int step, bool sleepy = false) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  if (!done) mm_wait_slow(bar, parity, dbg, code, step, sleepy);
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
      : "memory");
}

// 1-D bulk copy global -> shared (UBLKCP), completion signalled on an mbarrier; size and both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

}  // namespace amtk
