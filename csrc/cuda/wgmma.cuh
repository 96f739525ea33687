// Hopper warpgroup MMA (wgmma.mma_async, sm_90a) wrappers shared by the prefill GEMM and the prefill attention kernel.
// All shapes are m64n64k16 bf16 x bf16 -> f32: one warpgroup (128 threads) owns a 64 x 64 f32 accumulator, 32 registers a thread.
// Accumulator fragment of thread (warp w of the warpgroup, lane l), i = 0..7:
//   d[4i + 0, 1] = D[16w + l/4    ][8i + 2(l%4) + {0, 1}]
//   d[4i + 2, 3] = D[16w + l/4 + 8][8i + 2(l%4) + {0, 1}]
#pragma once
#include <cstdint>

namespace dl {

// Shared-memory matrix descriptor (sm_90 format) for a SWIZZLE_128B tile: rows of 128 B, 8-row groups 1024 B apart (stride byte
// offset). K-major tiles ignore the leading byte offset; MN-major tiles use it as the distance between 64-element atoms along M / N.
__device__ __forceinline__ uint64_t wgDesc(uint32_t smemAddr, uint32_t lboBytes = 16) {
    return (uint64_t)((smemAddr >> 4) & 0x3fffu) | ((uint64_t)((lboBytes >> 4) & 0x3fffu) << 16) | (64ull << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgFence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgCommit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgWait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Keeps the compiler from moving accumulator reads / writes across wgFence / wgWait.
__device__ __forceinline__ void wgFenceAcc(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D (+)= A . B, A [64 x 16] and B [16 x 64] from shared memory. B is K-major (stored [n][k]) unless TRANS_B (stored [k][n]).
template <int TRANS_B>
__device__ __forceinline__ void wgmmaSS(float (&d)[32], uint64_t descA, uint64_t descB, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(descA), "l"(descB), "r"(accumulate), "n"(TRANS_B));
}

// D (+)= A . B with A [64 x 16] bf16 in registers (the accumulator layout of a 64 x 16 tile, packed in pairs:
// a0 = rows l/4, cols 2(l%4)+{0,1}; a1 = rows l/4 + 8; a2 / a3 = the same rows, cols + 8) and B [16 x 64] MN-major in shared memory.
__device__ __forceinline__ void wgmmaRS(float (&d)[32], const uint32_t (&a)[4], uint64_t descB, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(descB), "r"(accumulate));
}

// Named barrier over the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads).
__device__ __forceinline__ void wgBarrier(uint32_t id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

}  // namespace dl
