// Shared device helpers for the sm_90a kernels: PTX wrappers (PDL, cache-hinted loads, mbarrier, TMA),
// warp reductions and the device weight layout description.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#define DL_EXPORT extern "C" __attribute__((visibility("default")))

#define DL_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess) {                                                                         \
            std::fprintf(stderr, "CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
                         cudaGetErrorString(_e));                                                        \
            return (int)_e;                                                                              \
        }                                                                                                \
    } while (0)

namespace dl {

// ---------------------------------------------------------------------------------------------------
// Device layout of a q40 matrix W[d][n] (quant blocks of 32 along n):
//   qs     : uint32 [d][n/8]   one word = 8 consecutive elements e0..e7, nibble i (bits 4i..4i+3) holds
//                              [e0,e2,e4,e6,e1,e3,e5,e7][i]  (value = nibble - 8)
//   scales : fp16   [d][n/32]
// Why this nibble order: (w >> 4s) & 0x000f000f yields the *adjacent* pair (e_{2s}, e_{2s+1}) in the two
// 16-bit halves — one LOP3 from a packed bf16x2 for the tensor-core path — while (w & 0x0f0f0f0f) and
// ((w>>4) & 0x0f0f0f0f) give byte quads for dp4a on the GEMV path. The file layout (reference
// src/nn/nn-quants.hpp:64-67: byte j = elem j | elem j+16 << 4, 18-byte blocks) is converted once at load.
// ---------------------------------------------------------------------------------------------------
struct Q40Matrix {
    const uint32_t *qs;
    const __half *scales;
    uint32_t d;   // rows
    uint32_t n;   // columns (elements)
};

constexpr int kWarp = 32;

__device__ __forceinline__ float warpSum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warpMax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- Programmatic dependent launch (PDL) ------------------------------------------------------------
// pdlLaunchDependents(): lets the next kernel in the stream start its prologue (weight prefetch) while this
// one is still running. pdlWait(): blocks until every prerequisite grid has completed and flushed.
__device__ __forceinline__ void pdlLaunchDependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdlWait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- cache-hinted global loads ----------------------------------------------------------------------
// Weights are streamed exactly once per token: bypass L1.
__device__ __forceinline__ uint4 ldgStream16(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint16_t ldgStreamU16(const void *p) {
    uint16_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ldgStreamU32(const void *p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

// ---- system-scope flag helpers for peer-memory signalling ------------------------------------------------
__device__ __forceinline__ void stReleaseSys(uint32_t *p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ldAcquireSys(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void stRelaxedSysF32(float *p, float v) {
    asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ float ldRelaxedSysF32(const float *p) {
    float v;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}

// LL ("low latency") words: 4 bytes of payload + a 4-byte valid flag travel in one 8-byte store, which the fabric
// delivers atomically — the receiver polls the word itself, no fence / separate flag round trip is needed.
__device__ __forceinline__ void stLL(uint64_t *p, uint32_t payload, uint32_t flag) {
    asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(payload), "r"(flag) : "memory");
}
__device__ __forceinline__ uint2 ldLL(const uint64_t *p) {
    uint2 v;
    asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ int dp4a(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));   // a: unsigned nibbles, b: signed int8
    return d;
}

// ---- in-kernel timeline (globaltimer ns) -----------------------------------------------------------------
// CTA 0 / thread 0 of every kernel stamps: [0] entry, [1] dependency resolved, [2] prologue done, [3] exit.
__device__ __forceinline__ uint64_t globalTimerNs() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void traceStamp(uint64_t *trace, int which) {
    if (trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0) trace[which] = globalTimerNs();
}

__device__ __forceinline__ float siluf(float x) { return x / (1.0f + __expf(-x)); }
// Gate activation of the feed-forward block, selected by the `.m` header's hidden_act (reference OP_SILU / OP_GELU,
// src/nn/nn-cpu-ops.cpp:454-500; gelu = tanh approximation). act: 0 = SiLU, 1 = GELU.
__device__ __forceinline__ float gateAct(float x, uint32_t act) {
    if (act == 0u) return siluf(x);
    const float u = 0.7978845608028654f * x * (1.0f + 0.044715f * x * x);
    return 0.5f * x * (1.0f + tanhf(u));
}

}  // namespace dl
