// Grid-barrier micro-benchmark (tools/microbench_barrier.py): the persistent decode kernel spends microseconds per software grid
// barrier, 5 barriers per layer. This kernel times candidate implementations under the same launch shape (one CTA per SM,
// 16 consumer warps + 1 producer warp, optional concurrent bulk-copy weight stream) so the choice is made on measurements.
#include "kernels.h"
#include "tma_common.cuh"

namespace dl {
namespace {

struct BarBenchArgs {
    unsigned int *ctr;        // [64][32] counters (one per 128-byte line)
    unsigned int *flags;      // [grid][32] per-CTA epoch words (one per 128-byte line)
    const uint8_t *stream;    // optional traffic source (>= 64 MB)
    uint64_t streamBytes;
    uint64_t *cycles;         // [grid] total ns per CTA
    uint32_t iters, variant, traffic, workNs;
};

__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }

__global__ void __launch_bounds__(kTmaThreads, 1) barBenchKernel(BarBenchArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + 4 * 36864);
    __shared__ volatile int stop;
    if (tid == 0) {
        for (int s = 0; s < 4; s++) mbarInit(&full[s], 1);
        stop = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == kConsumerWarps) {
        // traffic generator: back-to-back 36 KB bulk copies (what the weight producer does while the consumers sit in a barrier)
        if (lane == 0 && a.traffic) {
            const uint64_t policy = policyEvictFirst();
            uint64_t off = (uint64_t)blockIdx.x * 36864;
            uint32_t st = 0, par = 0;
            while (!stop) {
                mbarExpectTx(&full[st], 36864);
                tmaBulkLoad(smem + st * 36864, a.stream + off, 36864, &full[st], policy);
                off += (uint64_t)gridDim.x * 36864;
                if (off + 36864 > a.streamBytes) off = (uint64_t)blockIdx.x * 36864;
                mbarWait(&full[st], par);
                if (++st == 4) { st = 0; par ^= 1u; }
            }
        }
        return;
    }
    const uint32_t G = gridDim.x;
    unsigned int target = 0;
    uint32_t epoch = 0;
    const uint64_t t0 = globalTimerNs();
    for (uint32_t it = 0; it < a.iters; it++) {
        if (a.workNs) {   // staggered arrival: CTA-dependent busy wait
            const uint64_t w0 = globalTimerNs(), w = (uint64_t)a.workNs * ((blockIdx.x * 37u + it * 11u) % 16u) / 16u;
            while (globalTimerNs() - w0 < w) {}
        }
        epoch++;
        switch (a.variant) {
            case 0: {   // shipped: red.release + ld.acquire poll by one thread
                cbar();
                if (tid == 0) {
                    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.ctr) : "memory");
                    target += G;
                    unsigned int v;
                    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.ctr) : "memory"); } while (v < target);
                }
                cbar();
                break;
            }
            case 1: {   // relaxed arrive without any fence (NOT a correct barrier for data: measures the cost of the release)
                cbar();
                if (tid == 0) {
                    asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(a.ctr) : "memory");
                    target += G;
                    unsigned int v;
                    do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.ctr) : "memory"); } while (v < target);
                }
                cbar();
                break;
            }
            case 2: {   // per-CTA epoch flags, no atomics: thread 0 publishes, warp 0 polls all flags
                cbar();
                if (tid == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.flags + blockIdx.x * 32), "r"(epoch) : "memory");
                if (warp == 0) {
                    for (uint32_t c = lane; c < G; c += 32) {
                        unsigned int v;
                        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.flags + c * 32) : "memory"); } while ((int)(v - epoch) < 0);
                    }
                }
                cbar();
                break;
            }
            case 3: {   // 8 group counters on separate lines; 8 polling threads
                cbar();
                if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.ctr + (blockIdx.x & 7) * 32) : "memory");
                if (tid < 8) {
                    const unsigned int members = (G + 7 - tid) / 8;
                    const unsigned int tg = members * epoch;
                    unsigned int v;
                    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.ctr + tid * 32) : "memory"); } while (v < tg);
                }
                cbar();
                break;
            }
            case 4: {   // explicit fence + relaxed red, relaxed polls, acquire fence once at the end
                cbar();
                if (tid == 0) {
                    asm volatile("fence.acq_rel.gpu;" ::: "memory");
                    asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(a.ctr) : "memory");
                    target += G;
                    unsigned int v;
                    do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.ctr) : "memory"); } while (v < target);
                    asm volatile("fence.acq_rel.gpu;" ::: "memory");
                }
                cbar();
                break;
            }
            case 5: {   // flags written by all CTAs into ONE contiguous array (G words): warp 0 polls with 16-byte loads
                cbar();
                if (tid == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.flags + blockIdx.x), "r"(epoch) : "memory");
                if (warp == 0) {
                    for (uint32_t c = lane * 4; c < G; c += 128) {
                        uint4 v;
                        bool ok;
                        do {
                            asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(a.flags + c) : "memory");
                            ok = (int)(v.x - epoch) >= 0 && (c + 1 >= G || (int)(v.y - epoch) >= 0) && (c + 2 >= G || (int)(v.z - epoch) >= 0) &&
                                 (c + 3 >= G || (int)(v.w - epoch) >= 0);
                        } while (!ok);
                    }
                    asm volatile("fence.acq_rel.gpu;" ::: "memory");
                }
                cbar();
                break;
            }
            default: break;
        }
    }
    const uint64_t t1 = globalTimerNs();
    if (tid == 0) a.cycles[blockIdx.x] = t1 - t0;
    cbar();
    if (tid == 0) stop = 1;
}

}  // namespace
}  // namespace dl

DL_EXPORT int dl_bench_grid_barrier(int variant, uint32_t iters, int traffic, uint32_t workNs, unsigned int *ctr, unsigned int *flags,
                                    const void *stream, uint64_t streamBytes, uint64_t *nsOut, int grid, cudaStream_t s) {
    dl::BarBenchArgs a{};
    a.ctr = ctr; a.flags = flags; a.stream = (const uint8_t *)stream; a.streamBytes = streamBytes; a.cycles = nsOut;
    a.iters = iters; a.variant = (uint32_t)variant; a.traffic = (uint32_t)traffic; a.workNs = workNs;
    const size_t smem = 4 * 36864 + 64;
    static bool configured = false;
    if (!configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(dl::barBenchKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = true;
    }
    dl::barBenchKernel<<<grid, dl::kTmaThreads, smem, s>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}
