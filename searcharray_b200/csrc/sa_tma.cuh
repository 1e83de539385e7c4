// sa_tma.cuh -- 1-D bulk asynchronous copies (TMA, cp.async.bulk) + mbarrier helpers (sm_90a: Hopper TMA).
//
// Posting blocks are plain contiguous uint64 runs, so the 1-D bulk form of the Tensor Memory
// Accelerator is all that is needed: one elected thread arms an mbarrier with the byte count and
// issues `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes`; the copy engine moves
// the block into shared memory without occupying any thread's registers or issue slots, and every
// consumer thread waits on the barrier's phase bit.  (SASS: UBLKCP / SYNCS.ARRIVE.TRANS64 / SYNCS.)
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t sa_smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void sa_mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sa_smem_addr(bar)), "r"(count) : "memory");
}

// make the barrier initialisation visible to the async (TMA) proxy
__device__ __forceinline__ void sa_mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// generic-proxy writes/reads of a shared buffer must be ordered before the async proxy overwrites it
__device__ __forceinline__ void sa_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void sa_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa_smem_addr(bar)), "r"(bytes) : "memory");
}

// global -> shared bulk copy; dst, src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void sa_tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sa_smem_addr(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(sa_smem_addr(bar))
                 : "memory");
}

__device__ __forceinline__ void sa_mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(sa_smem_addr(bar)), "r"(phase)
        : "memory");
}

// Stages words[first, first + n) into shared memory with ONE bulk copy.  The global source must be
// 16-byte aligned for TMA while posting slices are only 8-byte aligned, so the copy starts at the
// aligned-down address and the caller reads the staged run at the returned offset (0 or 1 words).
// `dst` must be 16-byte aligned with room for n + 3 words; the source array must be readable for 2
// words past the slice (all index buffers carry pad words).  Returns the number of bytes requested
// (what the barrier has to expect); call from ONE thread after sa_mbar_expect_tx for the total.
__device__ __forceinline__ uint32_t sa_stage_bytes(const uint64_t *words, uint64_t first, uint32_t n) {
    const uint32_t head = (uint32_t)(((uintptr_t)(words + first) >> 3) & 1u);
    return ((n + head + 1u) & ~1u) * 8u;
}
__device__ __forceinline__ uint32_t sa_stage_issue(uint64_t *dst, const uint64_t *words, uint64_t first, uint32_t n, uint64_t *bar) {
    const uint32_t head = (uint32_t)(((uintptr_t)(words + first) >> 3) & 1u);
    const uint32_t bytes = ((n + head + 1u) & ~1u) * 8u;
    sa_tma_load_1d(dst, words + first - head, bytes, bar);
    return head;
}
#endif
