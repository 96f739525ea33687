// Shared device helpers of the TMA-fed GEMV kernels (gemv_q40_tma.cu, mega_decode.cu): mbarrier / bulk-copy PTX wrappers,
// consumer-warp barrier, warp reductions.
#pragma once
#include "kernels.h"

namespace dl {

constexpr int kConsumerWarps = 16;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kTmaThreads = kConsumerThreads + 32;
constexpr int kMaxStages = 16;
constexpr int kRowsPerStep = 4;

// ---- PTX wrappers ----
__device__ __forceinline__ uint32_t smemAddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbarInit(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarExpectTx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarArrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ void mbarWait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE;\n"
        "bra LAB_WAIT;\n"
        "LAB_DONE:\n"
        "}\n" ::"r"(smemAddr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ uint64_t policyEvictFirst() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policyEvictNormal() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void tmaBulkLoad(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smemAddr(dst)),
        "l"(src), "r"(bytes), "r"(smemAddr(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void consumerBarrier() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }

__device__ __forceinline__ float consumerSum(float v, float *red) {
    v = warpSum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    consumerBarrier();
    float t = (lane < kConsumerWarps) ? red[lane] : 0.f;
    t = warpSum(t);
    consumerBarrier();
    return t;
}

// Reduces 4 per-lane values over the warp; afterwards lane 8*i holds the total of value i.
__device__ __forceinline__ float reduce4(float v0, float v1, float v2, float v3, int lane) {
    const bool hi16 = lane & 16;
    float a = hi16 ? v2 : v0, b = hi16 ? v3 : v1;
    const float sa = hi16 ? v0 : v2, sb = hi16 ? v1 : v3;
    a += __shfl_xor_sync(0xffffffffu, sa, 16);
    b += __shfl_xor_sync(0xffffffffu, sb, 16);
    const bool hi8 = lane & 8;
    float c = hi8 ? b : a;
    const float sc = hi8 ? a : b;
    c += __shfl_xor_sync(0xffffffffu, sc, 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}

}  // namespace dl
