// Prefill GEMM on the Hopper tensor cores: out[T][d] = act_bf16[T][n] · dequant(W_q40[d][n])^T, T <= 256.
//
// Reference path replaced: batched OP_MATMUL via llamafile tinyBLAS (Q40×Q80 on CPU vector units,
// src/nn/nn-cpu-ops.cpp:1120-1136, src/nn/llamafile/sgemm.cpp:455-783) for the 32-token prefill chunks.
//
// sm_90a design (swap-AB: the 128 weight rows of a tile are the wgmma M dimension, two m64 halves; the tokens sit on N):
//   warp 0      TMA producer   — activations tile [64 tokens x 64 k] per stage via cp.async.bulk.tensor (SWIZZLE_128B)
//   warps 4-7   MMA + epilogue — one warpgroup issues 2 x 4 wgmma.mma_async (m64n64k16, bf16 -> f32 registers) per stage,
//                                releases the stage once the group before it has retired (wgmma.wait_group 1), and after the
//                                last stage runs the fused residual-add / SwiGLU / store epilogue from its registers
//   warps 8-15  dequant        — q40 nibbles + fp16 scale -> bf16, written straight into the canonical K-major
//                                SWIZZLE_128B wgmma tile in shared memory (generic proxy), fence.proxy.async, mbarrier arrive.
//                                This is the "q40 dequant fused into the GEMM prologue": the weights are never materialised
//                                in bf16 in global memory, HBM traffic stays at 4.5 bits/weight.
// A work item is one 128-row tile x one tile of up to 64 tokens (the f32 accumulator of 128 x 64 is 64 registers per consumer
// thread); chunks of more than 64 tokens are several token tiles of the same row tile, handled by neighbouring CTAs so the
// second read of the weights hits L2. Persistent CTAs loop over work items; all synchronisation is mbarrier based.
#include <cuda.h>
#include <cstdlib>

#include "kernels.h"
#include "wgmma.cuh"

namespace dl {

constexpr int kGmBlockM = 128;
constexpr int kGmBlockK = 64;
constexpr int kGmTokTile = 64;                 // tokens per work item = wgmma N
constexpr int kGmThreads = 512;
constexpr int kGmDeqWarps = 8;
constexpr int kGmMaxStages = 8;
constexpr int kGmMaxBStages = 12;
constexpr int kGmConsumerWarps = 4;
// accumulator staging for the epilogue: per consumer warp 32 rows x 16 tokens f32, row stride 17 (conflict-free row reads)
constexpr int kGmStgStride = 17;
constexpr int kGmStgBytes = kGmConsumerWarps * 32 * kGmStgStride * 4;
constexpr int kGmATileBytes = kGmBlockM * kGmBlockK * 2;   // 16 KB
constexpr int kGmBTileBytes = kGmTokTile * kGmBlockK * 2;  // 8 KB

enum { GEPI_STORE_F32 = 0, GEPI_RESIDUAL = 1, GEPI_SWIGLU_BF16 = 2 };

struct GemmArgs {
    const uint32_t *qs;
    const __half *scales;
    uint32_t d, n;        // weight rows / columns
    uint32_t T;           // tokens (grouped mode: the most tokens one group can have)
    void *out;
    uint32_t outStride;   // elements between tokens
    uint32_t stages;
    uint32_t bStages;      // TMA-staged variant: depth of the activation-tile ring (decoupled from the A-tile ring), in MMA steps
    uint32_t splitK;       // TMA-staged variant: K is cut into splitK ranges handled by different CTAs (work item = tile x split)
    float *splitScratch;   // [splitK][T][d] f32 partial accumulators
    uint32_t clusterSplit;  // TMA-staged variant: the splitK CTAs of a row tile form a thread-block cluster and reduce over distributed shared memory
    unsigned int *splitCounters;   // [row tiles x token tiles x 4][2], zero-initialised, self-resetting (arrived / done, per consumer warp)
    uint32_t rawStages;    // TMA-staged variant: depth of the raw q40 ring (2 or 3)
    uint32_t act;          // gate activation of GEPI_SWIGLU_BF16 (gHiddenAct)
    // Grouped (mixture-of-experts) mode, TMA-staged variant only: the weight matrix is nGroups stacked [grpRows][n] matrices, the
    // activation / output rows are sorted by group; group g owns rows [grpOffset[g], grpOffset[g] + grpCount[g]) (device arrays
    // written by moeSortKernel). Row tile t belongs to group t / grpTiles; token tiles without tokens are skipped by every warp role.
    const int *grpCount, *grpOffset;
    uint32_t grpTiles, grpRows, nGroups;
};

// ---- PTX wrappers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sAddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void gmBarInit(uint64_t *b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sAddr(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void gmBarExpectTx(uint64_t *b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sAddr(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gmBarArrive(uint64_t *b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sAddr(b)) : "memory"); }
__device__ __forceinline__ void gmBarWait(uint64_t *b, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nGM_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra GM_DONE;\nbra GM_WAIT;\nGM_DONE:\n}\n" ::"r"(sAddr(b)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tmaLoad2d(void *dst, const CUtensorMap *map, uint32_t c0, uint32_t c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(sAddr(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(sAddr(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// ---- thread-block cluster helpers (split-K reduce over distributed shared memory) ----
__device__ __forceinline__ uint32_t mapaShared(uint32_t localAddr, uint32_t ctaRank) {   // same offset in the peer CTA's shared memory
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(localAddr), "r"(ctaRank));
    return r;
}
__device__ __forceinline__ void stClusterF32(uint32_t clusterAddr, float v) { asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(clusterAddr), "f"(v) : "memory"); }
__device__ __forceinline__ void arriveRemote(uint32_t clusterAddr) {   // release at cluster scope: this thread's earlier DSMEM stores are visible to the waiter
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(clusterAddr) : "memory");
}
__device__ __forceinline__ void gmBarWaitCluster(uint64_t *b, uint32_t parity) {   // acquire at cluster scope (pairs with arriveRemote)
    uint32_t done = 0;
    while (true) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(sAddr(b)), "r"(parity) : "memory");
        if (done) break;
    }
}
__device__ __forceinline__ void clusterSync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- accumulator of one consumer warpgroup: rows [0, 64) in acc0, [64, 128) in acc1, 64 tokens ----------------------------
// The epilogue works row-wise: lane l of consumer warp q owns tile row gmRow(q, l) = 16q + (l & 15) + 64 (l >> 4), i.e. the 32 rows
// whose accumulator fragments the warp holds. gmLoadAcc transposes 16 token columns of those rows through the warp's staging
// buffer so every lane gets its row's 16 values.
__device__ __forceinline__ uint32_t gmRow(uint32_t q, uint32_t lane) { return 16u * q + (lane & 15u) + 64u * (lane >> 4); }

template <int CI>
__device__ __forceinline__ void gmStageSlab(float *stgW, const float (&acc)[32], uint32_t lane) {
    const uint32_t r = lane >> 2, c = 2u * (lane & 3u);
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
        const int i = 2 * CI + ii;   // 8-token column group of the fragment
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float *dst = stgW + (r + 8 * h) * kGmStgStride + ii * 8 + c;
            dst[0] = acc[4 * i + 2 * h];
            dst[1] = acc[4 * i + 2 * h + 1];
        }
    }
}
__device__ __forceinline__ void gmLoadAcc(float *stgW, const float (&acc0)[32], const float (&acc1)[32], uint32_t lane, uint32_t c0,
                                          uint32_t (&r)[16]) {
    __syncwarp();
    switch (c0 >> 4) {
        case 0: gmStageSlab<0>(stgW, acc0, lane); gmStageSlab<0>(stgW + 16 * kGmStgStride, acc1, lane); break;
        case 1: gmStageSlab<1>(stgW, acc0, lane); gmStageSlab<1>(stgW + 16 * kGmStgStride, acc1, lane); break;
        case 2: gmStageSlab<2>(stgW, acc0, lane); gmStageSlab<2>(stgW + 16 * kGmStgStride, acc1, lane); break;
        default: gmStageSlab<3>(stgW, acc0, lane); gmStageSlab<3>(stgW + 16 * kGmStgStride, acc1, lane); break;
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 16; j++) r[j] = __float_as_uint(stgW[lane * kGmStgStride + j]);
}

// ---- epilogue of one output element, shared by every reduce path -----------------------------------------------------------
// GEPI_RESIDUAL: the residual values of tokens [c0, c0 + N) (rows rowOff + c0 + j), all loaded before any store of the group so
// the read-modify-writes do not form a serialised chain. Tokens at or past `end` and features past the matrix read nothing.
template <int EPI, int N>
__device__ __forceinline__ void gmLoadResid(const GemmArgs &a, uint32_t rowOff, uint32_t c0, uint32_t end, uint32_t f, bool fOk,
                                            float (&resid)[N]) {
#pragma unroll
    for (int j = 0; j < N; j++)
        resid[j] = (EPI == GEPI_RESIDUAL && c0 + j < end && fOk) ? __ldcg(reinterpret_cast<const float *>(a.out) + (size_t)(rowOff + c0 + j) * a.outStride + f) : 0.f;
}
// Stores the finished value v of feature f into the output row starting at orow. Every lane of the warp calls it: SwiGLU pairs
// the gate (even row) with its up value (odd row, lane ^ 1) by a shuffle and the even lane stores the bf16 product.
template <int EPI>
__device__ __forceinline__ void gmStore(const GemmArgs &a, size_t orow, uint32_t f, float v, float resid, bool ok, uint32_t lane) {
    if (EPI == GEPI_SWIGLU_BF16) {
        const float other = __shfl_xor_sync(0xffffffffu, v, 1);   // rows (2i, 2i+1) = (gate_i, up_i)
        if (ok && !(lane & 1)) reinterpret_cast<__nv_bfloat16 *>(a.out)[orow + (f >> 1)] = __float2bfloat16_rn(gateAct(v, a.act) * other);
    } else if (ok) {
        reinterpret_cast<float *>(a.out)[orow + f] = EPI == GEPI_RESIDUAL ? v + resid : v;
    }
}

// One k-slice (64 wide) of the 128 x 64 tile: 4 x 2 wgmma (K = 16 each, +32 B per slice inside the swizzle atom; rows 64..127 of
// the A tile start 8 KB in).
__device__ __forceinline__ void gmMmaSlice(float (&acc0)[32], float (&acc1)[32], uint64_t descA, uint64_t descB, bool first) {
#pragma unroll
    for (uint32_t k = 0; k < kGmBlockK / 16; k++) {
        const uint32_t accum = (first && k == 0) ? 0u : 1u;
        wgmmaSS<0>(acc0, descA + 2 * k, descB + 2 * k, accum);
        wgmmaSS<0>(acc1, descA + (8192 >> 4) + 2 * k, descB + 2 * k, accum);
    }
}

template <int EPI>
__global__ void __launch_bounds__(kGmThreads, 1) gemmQ40TcKernel(const __grid_constant__ CUtensorMap tmapB, GemmArgs a) {
    extern __shared__ __align__(1024) uint8_t smemRaw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smemRaw) + 1023) & ~(uintptr_t)1023);
    // warp index through a shuffle: tells the compiler it is warp-uniform, so the role branches below are uniform control flow and
    // the wgmma / TMA operands (descriptors, barrier addresses) stay in uniform registers.
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const uint32_t stageBytes = kGmATileBytes + kGmBTileBytes;
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(smem + (size_t)a.stages * stageBytes);
    uint64_t *emptyBar = fullBar + kGmMaxStages;
    float *stg = reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(fullBar) + 512);

    const uint32_t nblk = a.n / 32;
    const uint32_t nkb = a.n / kGmBlockK;
    const uint32_t nTilesM = (a.d + kGmBlockM - 1) / kGmBlockM;
    const uint32_t nTT = (a.T + kGmTokTile - 1) / kGmTokTile;
    const uint32_t nItems = nTilesM * nTT;   // item = row tile x token tile

    pdlLaunchDependents();
    if (tid == 0) {
        for (uint32_t s = 0; s < a.stages; s++) {
            gmBarInit(&fullBar[s], 1 + kGmDeqWarps);
            gmBarInit(&emptyBar[s], kGmConsumerWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdlWait();   // activations (and the residual stream) come from the predecessor kernel

    if (warp == 0) {
        // ===================== TMA producer: activation tiles =====================
        if (lane == 0) {
            uint32_t it = 0;
            for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
                const uint32_t tok0 = (item % nTT) * kGmTokTile;
                for (uint32_t kb = 0; kb < nkb; kb++, it++) {
                    const uint32_t s = it % a.stages, ph = (it / a.stages) & 1;
                    gmBarWait(&emptyBar[s], ph ^ 1);
                    gmBarExpectTx(&fullBar[s], kGmBTileBytes);
                    tmaLoad2d(smem + (size_t)s * stageBytes + kGmATileBytes, &tmapB, kb * kGmBlockK, tok0, &fullBar[s]);
                }
            }
        }
    } else if (warp >= 4 && warp < 8) {
        // ===================== MMA + epilogue (one warpgroup) =====================
        const uint32_t q = warp - 4, row = gmRow(q, lane);
        float *stgW = stg + q * 32 * kGmStgStride;
        float acc0[32], acc1[32];
        uint32_t it = 0;
        for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
            const uint32_t tile = item / nTT, tok0 = (item % nTT) * kGmTokTile;
            const uint32_t Teff = min(a.T - tok0, (uint32_t)kGmTokTile);
            uint32_t prev = 0;
            for (uint32_t kb = 0; kb < nkb; kb++, it++) {
                const uint32_t s = it % a.stages, ph = (it / a.stages) & 1;
                gmBarWait(&fullBar[s], ph);
                const uint32_t aAddr = sAddr(smem + (size_t)s * stageBytes);
                wgFence();
                gmMmaSlice(acc0, acc1, wgDesc(aAddr), wgDesc(aAddr + kGmATileBytes), kb == 0);
                wgCommit();
                wgWait<1>();   // the stage before this one has been read by the tensor cores
                if (kb > 0) {
                    __syncwarp();
                    if (lane == 0) gmBarArrive(&emptyBar[prev]);
                }
                prev = s;
            }
            wgWait<0>();
            wgFenceAcc(acc0);
            wgFenceAcc(acc1);
            __syncwarp();
            if (lane == 0) gmBarArrive(&emptyBar[prev]);
            const uint32_t f = tile * kGmBlockM + row;     // output feature owned by this thread
            const bool fOk = f < a.d;
            for (uint32_t c0 = 0; c0 < Teff; c0 += 16) {
                uint32_t r[16];
                float resid[16];
                gmLoadResid<EPI>(a, tok0, c0, Teff, f, fOk, resid);
                gmLoadAcc(stgW, acc0, acc1, lane, c0, r);
#pragma unroll
                for (int j = 0; j < 16; j++)
                    gmStore<EPI>(a, (size_t)(tok0 + c0 + j) * a.outStride, f, __uint_as_float(r[j]), resid[j], c0 + j < Teff && fOk, lane);
            }
        }
    } else if (warp >= 8) {
        // ===================== dequant: q40 -> bf16 wgmma tile =====================
        const uint32_t dt = tid - 256;
        const uint32_t row = dt & 127, b = dt >> 7;                 // 128 rows x 2 quant blocks per 64-wide k slice
        const uint32_t swz = row & 7;
        uint32_t it = 0;
        for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
            const uint32_t tile = item / nTT;
            const uint32_t rowG = tile * kGmBlockM + row;
            const bool ok = rowG < a.d;
            const uint4 *qrow = reinterpret_cast<const uint4 *>(a.qs) + (size_t)rowG * nblk + b;
            const __half *srow = a.scales + (size_t)rowG * nblk + b;
            constexpr int G = 4;   // k-blocks per prefetch group
            uint4 curQ[G], nxtQ[G];
            uint16_t curS[G], nxtS[G];
            auto loadGroup = [&](uint32_t kb0, uint4 (&Q)[G], uint16_t (&S)[G]) {
#pragma unroll
                for (int g = 0; g < G; g++) {
                    const uint32_t kb = kb0 + g;
                    if (ok && kb < nkb) {
                        Q[g] = ldgStream16(qrow + (size_t)kb * 2);
                        S[g] = ldgStreamU16(srow + (size_t)kb * 2);
                    } else {
                        Q[g] = make_uint4(0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u);   // nibble 8 == value 0
                        S[g] = 0;
                    }
                }
            };
            loadGroup(0, curQ, curS);
            for (uint32_t kb0 = 0; kb0 < nkb; kb0 += G) {
                if (kb0 + G < nkb) loadGroup(kb0 + G, nxtQ, nxtS);
#pragma unroll
                for (int g = 0; g < G; g++) {
                    const uint32_t kb = kb0 + g;
                    if (kb < nkb) {
                        const uint32_t s = it % a.stages, ph = (it / a.stages) & 1;
                        gmBarWait(&emptyBar[s], ph ^ 1);
                        uint8_t *aTile = smem + (size_t)s * stageBytes;
                        const __nv_bfloat16 sc = __float2bfloat16_rn(__half2float(__ushort_as_half(curS[g])));
                        const __nv_bfloat162 sc2 = __halves2bfloat162(sc, sc);
                        const __nv_bfloat162 off = __floats2bfloat162_rn(136.f, 136.f);
                        const uint32_t w[4] = {curQ[g].x, curQ[g].y, curQ[g].z, curQ[g].w};
#pragma unroll
                        for (int c = 0; c < 4; c++) {
                            uint32_t o[4];
#pragma unroll
                            for (int sft = 0; sft < 4; sft++) {
                                // (nibble | 0x4300) is the bf16 value 128 + nibble; subtract 136 -> nibble - 8 (exact), then scale
                                uint32_t t = ((w[c] >> (4 * sft)) & 0x000f000fu) | 0x43004300u;
                                __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162 *>(&t);
                                v = __hmul2(__hsub2(v, off), sc2);
                                o[sft] = *reinterpret_cast<uint32_t *>(&v);
                            }
                            const uint32_t chunk = (b * 4 + c) ^ swz;                       // SWIZZLE_128B: 16-byte chunk index XOR (row % 8)
                            *reinterpret_cast<uint4 *>(aTile + row * 128 + chunk * 16) = make_uint4(o[0], o[1], o[2], o[3]);
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> visible to the tensor core
                        __syncwarp();
                        if (lane == 0) gmBarArrive(&fullBar[s]);
                        it++;
                    }
                }
#pragma unroll
                for (int g = 0; g < G; g++) { curQ[g] = nxtQ[g]; curS[g] = nxtS[g]; }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Variant with the raw q40 stream staged by TMA (n % 256 == 0): warp 3 issues two tensor-map loads per 256-wide K chunk
// ([128 rows x 128 B] nibbles, SWIZZLE_128B so the 16-byte reads of 8 consecutive rows hit different banks, and
// [128 rows x 16 B] scales) into a 3-deep ring; the dequant warps read the chunk from shared memory. ~54 KB of weight
// bytes are in flight per SM instead of the 16 KB the register-prefetching variant above can hold.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kGmRawStagesMax = 8;
constexpr int kGmRawK = 256;
constexpr int kGmRawQsBytes = kGmBlockM * 128;               // 16 KB
constexpr int kGmRawStageBytes = kGmRawQsBytes + kGmBlockM * 16;   // + 2 KB scales

template <int EPI>
__global__ void __launch_bounds__(kGmThreads, 1) gemmQ40TcTmaKernel(const __grid_constant__ CUtensorMap tmapB,
                                                                    const __grid_constant__ CUtensorMap tmapQ,
                                                                    const __grid_constant__ CUtensorMap tmapS, GemmArgs a) {
    extern __shared__ __align__(1024) uint8_t smemRaw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smemRaw) + 1023) & ~(uintptr_t)1023);
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // see gemmQ40TcKernel
    // Two independent rings: A tiles (dequantised weights, written by the dequant warps) and B tiles (activations, TMA). With one
    // combined stage only one A tile per dequant group fits, so every group would wait for the MMA of its previous tile before
    // converting the next; the A ring is 8 deep (2 per group) where shared memory allows.
    uint8_t *bBase = smem + (size_t)a.stages * kGmATileBytes;
    uint8_t *rawBase = bBase + (size_t)a.bStages * kGmBTileBytes;        // [rawStages][18 KB], 1024-aligned (all tiles are multiples of 1 KB)
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(rawBase + (size_t)a.rawStages * kGmRawStageBytes);   // A tile converted
    uint64_t *emptyBar = fullBar + kGmMaxStages;                                                            // A tile consumed
    uint64_t *bFull = emptyBar + kGmMaxStages;
    uint64_t *rawFull = bFull + kGmMaxBStages;
    uint64_t *rawEmpty = rawFull + kGmRawStagesMax;
    uint64_t *freeBar = rawEmpty + kGmRawStagesMax;   // [4 source ranks][4 consumer warps]: "the rings of rank r are free" (cluster split-K)
    uint64_t *dataBar = freeBar + 16;                 // [4 consumer warps]: every peer has delivered its partial sums for my tokens
    float *stg = reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(fullBar) + 1024);

    const uint32_t nkb = a.n / kGmBlockK;
    const uint32_t nkq = (a.n + kGmRawK - 1) / kGmRawK;
    const uint32_t nTilesM = a.grpCount ? a.nGroups * a.grpTiles : (a.d + kGmBlockM - 1) / kGmBlockM;
    const uint32_t nTT = (a.T + kGmTokTile - 1) / kGmTokTile;
    const uint32_t splitK = a.splitK;
    const uint32_t nItems = nTilesM * nTT * splitK;
    // work item -> (row tile, token tile, K range in 256-wide raw chunks); consecutive items share a row tile
    auto kqBegin = [&](uint32_t ks) { return (uint32_t)(((uint64_t)ks * nkq) / splitK); };
    auto itemTile = [&](uint32_t item) { return item / (splitK * nTT); };
    auto itemTT = [&](uint32_t item) { return (item / splitK) % nTT; };
    // a.stages is 4 or 8 (tmaGeometry): stage / phase of the A ring by shift and mask; the raw and B rings (arbitrary depth) keep
    // incremental (stage, parity) counters — a runtime `%` or `/` is a ~25-instruction I2F/MUFU.RCP sequence per use
    const uint32_t aMask = a.stages - 1, aShift = a.stages == 8 ? 3u : 2u;
    const bool grouped = a.grpCount != nullptr;
    // grouped mode: (tile) -> weight row of the tile's first row; (tile, token tile) -> first activation/output row, valid tokens
    auto tileRow0 = [&](uint32_t tile) { return grouped ? (tile / a.grpTiles) * a.grpRows + (tile % a.grpTiles) * kGmBlockM : tile * kGmBlockM; };
    auto tileTokens = [&](uint32_t tile, uint32_t tt) -> uint32_t {
        const uint32_t total = grouped ? (uint32_t)__ldg(a.grpCount + tile / a.grpTiles) : a.T, t0 = tt * kGmTokTile;
        return total > t0 ? min(total - t0, (uint32_t)kGmTokTile) : 0u;
    };
    auto tileTok0 = [&](uint32_t tile, uint32_t tt) { return (grouped ? (uint32_t)__ldg(a.grpOffset + tile / a.grpTiles) : 0u) + tt * kGmTokTile; };

    pdlLaunchDependents();
    if (tid == 0) {
        for (uint32_t s = 0; s < a.stages; s++) {
            gmBarInit(&fullBar[s], 2);   // the two dequant warps of the group that fills the slice
            gmBarInit(&emptyBar[s], kGmConsumerWarps);
        }
        for (uint32_t s = 0; s < a.bStages; s++) gmBarInit(&bFull[s], 1);
        for (uint32_t i = 0; i < a.rawStages; i++) {
            gmBarInit(&rawFull[i], 1);
            gmBarInit(&rawEmpty[i], kGmDeqWarps);
        }
        if (a.clusterSplit) {
            for (int i = 0; i < 16; i++) gmBarInit(&freeBar[i], 1);
            for (int i = 0; i < 4; i++) gmBarInit(&dataBar[i], (a.splitK - 1) * 32);   // every lane of the peers' warp q arrives after its stores
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (a.clusterSplit) clusterSync();   // no peer may arrive on (or write into) this CTA before its barriers exist

    if (warp == 3) {
        // ===================== raw weight producer (weights are constants: no dependency wait) =====================
        if (lane == 0) {
            uint32_t rs = 0, ph = 0;
            for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
                const uint32_t tile = itemTile(item), ks = item % splitK;
                if (tileTokens(tile, itemTT(item)) == 0) continue;
                const uint32_t wRow = tileRow0(tile);
                for (uint32_t kq = kqBegin(ks); kq < kqBegin(ks + 1); kq++) {
                    gmBarWait(&rawEmpty[rs], ph ^ 1);
                    uint8_t *dst = rawBase + (size_t)rs * kGmRawStageBytes;
                    gmBarExpectTx(&rawFull[rs], kGmRawStageBytes);
                    tmaLoad2d(dst, &tmapQ, kq * 128, wRow, &rawFull[rs]);                 // nibbles: 128 B per row
                    tmaLoad2d(dst + kGmRawQsBytes, &tmapS, kq * 16, wRow, &rawFull[rs]);   // scales: 16 B per row
                    if (++rs == a.rawStages) { rs = 0; ph ^= 1u; }
                }
            }
        }
    } else if (warp == 0) {
        // ===================== activation producer =====================
        pdlWait();
        if (lane == 0) {
            uint32_t it = 0, sbP = 0;
            for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
                const uint32_t ks = item % splitK, tile = itemTile(item), tt = itemTT(item);
                if (tileTokens(tile, tt) == 0) continue;
                const uint32_t tok0 = tileTok0(tile, tt);
                for (uint32_t kb = kqBegin(ks) * 4; kb < min(kqBegin(ks + 1) * 4, nkb); kb++, it++) {
                    // `it` counts k-slices. B stage s was last read by the MMAs of slice it - bStages; their completion is already
                    // signalled on the A ring's emptyBar. bStages <= stages, so that phase cannot have been overtaken.
                    const uint32_t s = sbP;
                    if (it >= a.bStages) {
                        const uint32_t j = it - a.bStages;
                        gmBarWait(&emptyBar[j & aMask], (j >> aShift) & 1);
                    }
                    gmBarExpectTx(&bFull[s], kGmBTileBytes);
                    tmaLoad2d(bBase + (size_t)s * kGmBTileBytes, &tmapB, kb * kGmBlockK, tok0, &bFull[s]);
                    if (++sbP == a.bStages) sbP = 0;
                }
            }
        }
    } else if (warp >= 4 && warp < 8) {
        // ===================== MMA + epilogue (one warpgroup) =====================
        pdlWait();   // the residual stream is read-modify-written
        const uint32_t q = warp - 4, row = gmRow(q, lane);
        float *stgW = stg + q * 32 * kGmStgStride;
        float acc0[32], acc1[32];
        auto loadAcc = [&](uint32_t c0, uint32_t (&r)[16]) { gmLoadAcc(stgW, acc0, acc1, lane, c0, r); };
        uint32_t itBase = 0, sbM = 0, phbM = 0;
        for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
            const uint32_t ks = item % splitK, tile = itemTile(item), tt = itemTT(item);
            const uint32_t Teff = tileTokens(tile, tt);
            if (Teff == 0) continue;
            const uint32_t kb0 = kqBegin(ks) * 4, kb1 = min(kqBegin(ks + 1) * 4, nkb);
            uint32_t prevSlot = 0;
            for (uint32_t kb = kb0; kb < kb1; kb++) {
                const uint32_t it = itBase + (kb - kb0);                 // k-slice counter of the step's first slice
                const uint32_t s = it & aMask, ph = (it >> aShift) & 1;
                const uint32_t sb = sbM, phb = phbM;
                if (++sbM == a.bStages) { sbM = 0; phbM ^= 1u; }
                gmBarWait(&bFull[sb], phb);
                gmBarWait(&fullBar[s], ph);
                const uint64_t descA = wgDesc(sAddr(smem + (size_t)s * kGmATileBytes));
                const uint64_t descB = wgDesc(sAddr(bBase + (size_t)sb * kGmBTileBytes));
                wgFence();
                gmMmaSlice(acc0, acc1, descA, descB, kb == kb0);
                wgCommit();
                wgWait<1>();   // the previous slice's tiles have been read by the tensor cores: release them
                if (kb != kb0) {
                    __syncwarp();
                    if (lane == 0) gmBarArrive(&emptyBar[prevSlot]);
                }
                prevSlot = s;
            }
            wgWait<0>();
            wgFenceAcc(acc0);
            wgFenceAcc(acc1);
            __syncwarp();
            if (lane == 0) gmBarArrive(&emptyBar[prevSlot]);
            itBase += kb1 - kb0;
            // grouped mode: f is the feature index inside the group's matrix, output rows start at the group's first sorted row
            const uint32_t f = (grouped ? (tile % a.grpTiles) * kGmBlockM : tile * kGmBlockM) + row;
            const bool fOk = f < (grouped ? a.grpRows : a.d);
            const uint32_t rowOff = tileTok0(tile, tt);
            if (splitK > 1 && a.clusterSplit) {
                // ---- split-K inside a thread-block cluster: the splitK CTAs of this work item are the ranks of one cluster (rank = ks).
                // Rank r reduces the tokens [r * per, (r + 1) * per): every other rank stores its partial sums for those tokens
                // straight into r's shared memory (st.shared::cluster into the A ring, which is idle once r's accumulator is
                // complete) and arrives on r's mbarrier; r adds them in rank order (deterministic) to its own accumulator columns and
                // runs the epilogue. No global scratch, no MEMBAR.GPU, no atomics: two DSMEM hops instead of three L2 round trips.
                const uint32_t per = ((Teff + splitK - 1) / splitK + 15u) & ~15u;     // 16-token granularity = one gmLoadAcc
                const uint32_t recvLocal = sAddr(smem);                                // float recv[splitK - 1][per][128] in the A ring
                if (lane == 0)
                    for (uint32_t p = 0; p < splitK; p++)
                        if (p != ks) arriveRemote(mapaShared(sAddr(&freeBar[ks * 4 + q]), p));   // my MMAs are done: my rings may be overwritten
                for (uint32_t dp = 1; dp < splitK; dp++) {
                    const uint32_t p = (ks + dp) % splitK;                             // staggered order: not everybody hits rank 0 first
                    const uint32_t pBeg = p * per, pEnd = min(Teff, pBeg + per);
                    gmBarWaitCluster(&freeBar[p * 4 + q], 0);
                    const uint32_t slot = ks < p ? ks : ks - 1;                        // my place among p's splitK - 1 sources, in rank order
                    const uint32_t dstBase = mapaShared(recvLocal + (slot * per * kGmBlockM + row) * 4u, p);
                    for (uint32_t c0 = pBeg; c0 < pEnd; c0 += 16) {
                        uint32_t r[16];
                        loadAcc(c0, r);
#pragma unroll
                        for (int j = 0; j < 16; j++)
                            if (c0 + j < pEnd) stClusterF32(dstBase + (c0 + j - pBeg) * (kGmBlockM * 4u), __uint_as_float(r[j]));
                    }
                    arriveRemote(mapaShared(sAddr(&dataBar[q]), p));                   // every lane: its own stores are released
                }
                const uint32_t tBeg = ks * per, tEnd = min(Teff, tBeg + per);
                gmBarWaitCluster(&dataBar[q], 0);
                const float *recv = reinterpret_cast<const float *>(smem);
                for (uint32_t c0 = tBeg; c0 < tEnd; c0 += 16) {
                    uint32_t own[16];
                    loadAcc(c0, own);
                    float resid[16];
                    gmLoadResid<EPI>(a, rowOff, c0, tEnd, f, fOk, resid);
#pragma unroll
                    for (int j = 0; j < 16; j++) {
                        const uint32_t tok = c0 + j;
                        float v = 0.f;
                        for (uint32_t r = 0; r < splitK; r++) {                        // rank order, own partial at position ks
                            if (r == ks) v += __uint_as_float(own[j]);
                            else if (tok < tEnd) v += recv[(((r < ks ? r : r - 1) * per) + (tok - tBeg)) * kGmBlockM + row];
                        }
                        gmStore<EPI>(a, (size_t)(rowOff + tok) * a.outStride, f, v, resid[j], fOk && tok < tEnd, lane);
                    }
                }
                continue;
            }
            if (splitK > 1) {
                // ---- split-K: park the partial accumulator; once all splits of this warp's 32 rows have arrived, every split reduces
                // its own share of the tokens (fixed summation order -> deterministic). All splits of a work item are co-resident
                // (one item per CTA, nItems <= SMs), so the wait cannot deadlock; the reduce is latency-bound (a dependent L2 round
                // trip per round of 8 tokens), which is why it is spread over the splits instead of left to the last arriver.
                float *mineS = a.splitScratch + (size_t)ks * a.T * a.d;
                for (uint32_t c0 = 0; c0 < Teff; c0 += 16) {
                    uint32_t r[16];
                    loadAcc(c0, r);
#pragma unroll
                    for (int j = 0; j < 16; j++)
                        if (c0 + j < Teff && fOk) mineS[(size_t)(rowOff + c0 + j) * a.d + f] = __uint_as_float(r[j]);
                }
                __threadfence();
                __syncwarp();
                unsigned int *ctr = a.splitCounters + (size_t)((tile * nTT + tt) * 4 + q) * 2;   // [0]: splits arrived, [1]: splits done reducing
                if (lane == 0) {
                    atomicAdd(ctr, 1u);
                    unsigned int seen = 0, spins = 0;
                    do {
                        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctr) : "memory");
                        if (seen < splitK) __nanosleep(64);
                    } while (seen < splitK && ++spins < (1u << 24));
                }
                __syncwarp();
                const uint32_t per = (Teff + splitK - 1) / splitK, tBeg = ks * per, tEnd = min(Teff, tBeg + per);
                for (uint32_t tok0 = tBeg; tok0 < tEnd; tok0 += 8) {
                    // 8 tokens x up to 4 splits (+ 8 residual values) are loaded before any arithmetic: ~40 loads in flight per thread
                    float part[8][4], res[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const bool ok = fOk && tok0 + j < tEnd;
#pragma unroll
                        for (int k2 = 0; k2 < 4; k2++)
                            part[j][k2] = (ok && (uint32_t)k2 < splitK) ? __ldcg(a.splitScratch + ((size_t)k2 * a.T + rowOff + tok0 + j) * a.d + f) : 0.f;
                    }
                    gmLoadResid<EPI>(a, rowOff, tok0, tEnd, f, fOk, res);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const uint32_t tok = tok0 + j;
                        float v = 0.f;
#pragma unroll
                        for (int k2 = 0; k2 < 4; k2++) v += part[j][k2];          // fixed order -> deterministic
                        gmStore<EPI>(a, (size_t)(rowOff + tok) * a.outStride, f, v, res[j], fOk && tok < tEnd, lane);
                    }
                }
                __syncwarp();
                if (lane == 0) {
                    // the split that finishes last re-arms the counters for the next launch (everyone has passed the wait by then)
                    if (atomicAdd(ctr + 1, 1u) == splitK - 1) { ctr[0] = 0; ctr[1] = 0; }
                }
                continue;
            }
            for (uint32_t c0 = 0; c0 < Teff; c0 += 16) {
                uint32_t r[16];
                float resid[16];
                gmLoadResid<EPI>(a, rowOff, c0, Teff, f, fOk, resid);
                loadAcc(c0, r);
#pragma unroll
                for (int j = 0; j < 16; j++)
                    gmStore<EPI>(a, (size_t)(rowOff + c0 + j) * a.outStride, f, __uint_as_float(r[j]), resid[j], c0 + j < Teff && fOk, lane);
            }
        }
    } else if (warp >= 8) {
        // ===================== dequant: shared-memory q40 chunk -> bf16 wgmma tile =====================
        // Four groups of two warps; group g converts the g-th 64-wide k-slice of every 256-wide raw chunk, so four A tiles
        // are being converted concurrently and the load -> convert -> store -> proxy-fence latency of one slice overlaps
        // with the others (one group per slice instead of all eight warps serialising on every slice).
        const uint32_t grp = (uint32_t)(warp - 8) >> 1;
        const uint32_t j = (uint32_t)tid - 256u - grp * 64u;       // 0..63: rows j and j + 64
        const __nv_bfloat162 off = __floats2bfloat162_rn(136.f, 136.f);
        uint32_t nibMask = 0x000f000fu, bfMagic = 0x43004300u;
        asm volatile("" : "+r"(nibMask), "+r"(bfMagic));   // opaque: keeps both constants in registers
        uint32_t itR = 0, rsD = 0, rphD = 0;
        for (uint32_t item = blockIdx.x; item < nItems; item += gridDim.x) {
            const uint32_t ks = item % splitK;
            if (tileTokens(itemTile(item), itemTT(item)) == 0) continue;
            for (uint32_t kq = kqBegin(ks); kq < kqBegin(ks + 1); kq++, itR++) {
                const uint32_t rs = rsD, rph = rphD;
                if (++rsD == a.rawStages) { rsD = 0; rphD ^= 1u; }
                gmBarWait(&rawFull[rs], rph);
                const uint8_t *rbase = rawBase + (size_t)rs * kGmRawStageBytes;
                uint4 qv[2][2];
                uint16_t sv[2][2];
#pragma unroll
                for (int rr = 0; rr < 2; rr++) {
                    const uint32_t row = j + 64 * rr;
#pragma unroll
                    for (int b = 0; b < 2; b++) {
                        const uint32_t c8 = grp * 2 + b;
                        qv[rr][b] = *reinterpret_cast<const uint4 *>(rbase + row * 128 + ((c8 ^ (row & 7)) << 4));
                        sv[rr][b] = *reinterpret_cast<const uint16_t *>(rbase + kGmRawQsBytes + row * 16 + c8 * 2);
                    }
                }
                // the raw chunk now lives in registers: hand the stage back to the TMA producer before the (long) conversion
                __syncwarp();
                if (lane == 0) gmBarArrive(&rawEmpty[rs]);
                const uint32_t itA = itR * 4 + grp;
                const uint32_t s = itA & aMask, ph = (itA >> aShift) & 1;
                gmBarWait(&emptyBar[s], ph ^ 1);
                uint8_t *aTile = smem + (size_t)s * kGmATileBytes;
#pragma unroll
                for (int rr = 0; rr < 2; rr++) {
                    const uint32_t row = j + 64 * rr;
                    const uint32_t swz = row & 7;
#pragma unroll
                    for (int b = 0; b < 2; b++) {
                        const __nv_bfloat16 sc = __float2bfloat16_rn(__half2float(__ushort_as_half(sv[rr][b])));
                        const __nv_bfloat162 sc2 = __halves2bfloat162(sc, sc);
                        const uint32_t w[4] = {qv[rr][b].x, qv[rr][b].y, qv[rr][b].z, qv[rr][b].w};
#pragma unroll
                        for (int c = 0; c < 4; c++) {
                            uint32_t o[4];
#pragma unroll
                            for (int sft = 0; sft < 4; sft++) {
                                // (x & 0x000f000f) | 0x43004300 as ONE lop3 (both constants in registers; with immediates the
                                // compiler emits two LOP3 per pair: the conversion is issue-bound, ~4.75 -> 3.75 instructions per pair)
                                uint32_t t;
                                asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(t) : "r"(w[c] >> (4 * sft)), "r"(nibMask), "r"(bfMagic));
                                __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162 *>(&t);
                                v = __hmul2(__hsub2(v, off), sc2);
                                o[sft] = *reinterpret_cast<uint32_t *>(&v);
                            }
                            const uint32_t chunk = (uint32_t)(b * 4 + c) ^ swz;
                            *reinterpret_cast<uint4 *>(aTile + row * 128 + chunk * 16) = make_uint4(o[0], o[1], o[2], o[3]);
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) gmBarArrive(&fullBar[s]);
            }
        }
    }
}

// ---- host side -----------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encodeTiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

template <int EPI>
static int launchGemm(const CUtensorMap &mapB, const CUtensorMap *mapQ, const CUtensorMap *mapS, const GemmArgs &a, int grid,
                      size_t smemBytes, cudaStream_t stream, bool pdl) {
    static size_t configured[2] = {0, 0};
    const int variant = mapQ ? 1 : 0;
    if (smemBytes > configured[variant]) {
        if (variant) DL_CUDA_CHECK(cudaFuncSetAttribute(gemmQ40TcTmaKernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
        else DL_CUDA_CHECK(cudaFuncSetAttribute(gemmQ40TcKernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
        configured[variant] = smemBytes;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kGmThreads);
    cfg.dynamicSmemBytes = smemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (variant && a.clusterSplit) {   // the splitK CTAs of a row tile = one cluster (consecutive blockIdx.x), reduce over DSMEM
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = a.splitK; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
        cfg.numAttrs = 2;
    }
    if (variant) DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gemmQ40TcTmaKernel<EPI>, mapB, *mapQ, *mapS, a));
    else DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gemmQ40TcKernel<EPI>, mapB, a));
    return 0;
}

static bool encode2d(EncodeTiledFn enc, CUtensorMap *map, CUtensorMapDataType type, const void *base, uint64_t inner, uint64_t outer,
                     uint64_t strideBytes, uint32_t boxInner, uint32_t boxOuter, CUtensorMapSwizzle swz) {
    const cuuint64_t dims[2] = {inner, outer};
    const cuuint64_t strides[1] = {strideBytes};
    const cuuint32_t box[2] = {boxInner, boxOuter};
    const cuuint32_t estr[2] = {1, 1};
    return enc(map, type, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Shared-memory geometry of the TMA-staged variant: A ring (multiple of 4: each dequant group always revisits its own stages),
// B ring (>= 2 activation tiles), raw q40 ring. Returns the dynamic shared-memory size, 0 if nothing fits.
static size_t tmaGeometry(GemmArgs &a) {
    const size_t bTile = kGmBTileBytes;
    const size_t budget = 227 * 1024 - 1024 - 1024 - kGmStgBytes;   // 1 KB alignment slack + 1 KB of mbarriers + epilogue staging
    // Candidates in order of preference: {A slices, raw stages, minimum B slices}: the deeper A ring (two slices per dequant group)
    // first, then >= 4 k-slices of activations in flight.
    static const uint32_t cand[6][3] = {{8, 3, 4}, {8, 2, 4}, {4, 3, 4}, {4, 2, 4}, {8, 2, 2}, {4, 2, 2}};
    for (int i = 0; i < 6; i++) {
        const uint32_t nA = cand[i][0], nRaw = cand[i][1], minB = cand[i][2];
        const size_t fixed = (size_t)nA * kGmATileBytes + (size_t)nRaw * kGmRawStageBytes;
        if (fixed + minB * bTile > budget) continue;
        size_t nb = (budget - fixed) / bTile;
        if (nb > 4) nb = 4;      // released through the A ring's barriers: never deeper than it
        a.stages = nA; a.rawStages = nRaw; a.bStages = (uint32_t)nb;
        return fixed + nb * bTile + 1024 + 1024 + kGmStgBytes;
    }
    return 0;
}

// Dispatch decision of gemmQ40TcV: kernel, shared-memory geometry, split-K and reduce scheme, grid. Pure host code (reads only the
// DL_GEMM_CLUSTER / DL_GEMM_SPLITK switches), so dl_gemm_q40_tc_plan can report what a launch with the same
// arguments runs. rc != 0: the launcher's return code for a shape it does not cover.
struct GemmPlan {
    int rc;
    bool tma;              // TMA-staged variant (else the register-prefetch one)
    uint32_t stages, rawStages, bStages, splitK, clusterSplit, grid;
    size_t smemBytes;
};

static GemmPlan planGemmQ40Tc(int epi, uint32_t d, uint32_t n, uint32_t T, uint32_t actStride, int numSms, int variant) {
    GemmPlan p{};
    p.rc = -1;
    if (T == 0 || T > 256 || n % kGmBlockK || d % 2) return p;
    p.rc = -6;
    p.tma = variant == 2 || (variant == 0 && n % 256 == 0);
    if (p.tma && n % 256) return p;
    p.rc = -4;
    if (actStride % 8) return p;   // the activation tensor map needs a row pitch that is a multiple of 16 bytes
    const size_t stageBytes = kGmATileBytes + kGmBTileBytes;
    const size_t budget = 227 * 1024 - 1024 - 512 - kGmStgBytes;
    if (p.tma) {
        GemmArgs g{};
        p.smemBytes = tmaGeometry(g);
        if (!p.smemBytes) {
            p.rc = -9;
            if (variant == 2) return p;
            p.tma = false;
        } else {
            p.stages = g.stages; p.rawStages = g.rawStages; p.bStages = g.bStages;
        }
    }
    if (!p.tma) {
        p.stages = (uint32_t)(budget / stageBytes);
        if (p.stages > (uint32_t)kGmMaxStages) p.stages = kGmMaxStages;
        p.rc = -3;
        if (p.stages < 2) return p;
        p.smemBytes = p.stages * stageBytes + 1024 + 512 + kGmStgBytes;
    }
    p.rc = -5;
    if (epi < GEPI_STORE_F32 || epi > GEPI_SWIGLU_BF16) return p;
    p.rc = 0;
    const uint32_t nTilesM = (d + kGmBlockM - 1) / kGmBlockM;
    const uint32_t nTT = (T + kGmTokTile - 1) / kGmTokTile;
    p.splitK = 1;
    if (p.tma) {
        // small-d matrices (qkv, wo, w2) leave most SMs idle with one CTA per work item: cut K so that ~all SMs get an item
        const uint32_t nkq = n / 256;
        uint32_t sk = (uint32_t)numSms / (nTilesM * nTT);
        // The k-loop of one CTA is latency-bound, so idle SMs are worth a split even at K = 4096; the cooperative reduce costs a
        // few us. At most 4 splits (reduce register budget), every split keeps >= 4 raw chunks (1024 of K), and all items must be
        // co-resident (the reduce waits for its sibling splits).
        if (sk > 4) sk = 4;
        if (sk > nkq / 4) sk = nkq / 4;
        // reduce over distributed shared memory (thread-block cluster) when the receive buffer ((sk - 1) x per x 128 f32) fits into the
        // idle A ring: two DSMEM hops instead of the global-scratch round trips
        const char *clEnv = getenv("DL_GEMM_CLUSTER");
        auto clusterFits = [&](uint32_t k) {
            const uint32_t per = ((min(T, (uint32_t)kGmTokTile) + k - 1) / k + 15u) & ~15u;
            // clusters of 2 or 4 only (a power of two divides the GPC evenly)
            return (k == 2 || k == 4) && (size_t)(k - 1) * per * kGmBlockM * 4 <= (size_t)p.stages * kGmATileBytes && !(clEnv && clEnv[0] == '0');
        };
        // K < 8192 with fewer than 4 splits does not pay for the reduce
        if (nkq < 32 && sk < 4) sk = 1;
        if (const char *f = getenv("DL_GEMM_SPLITK")) { const uint32_t want = (uint32_t)atoi(f); if (want >= 1 && want < sk) sk = want; }
        if (sk >= 2 && nTilesM * nTT * 8 <= 4096) {
            p.splitK = sk;
            p.clusterSplit = clusterFits(sk) ? 1u : 0u;
        }
    }
    const uint32_t nItems = nTilesM * nTT * p.splitK;
    p.grid = nItems < (uint32_t)numSms ? nItems : (uint32_t)numSms;
    return p;
}

// act: bf16 [T][n] row-major (row stride actStride elements). variant: 0 auto, 1 register-prefetch dequant, 2 TMA-staged raw weights.
static float *gSplitScratch = nullptr;
static unsigned int *gSplitCounters = nullptr;
static size_t gSplitScratchBytes = 0;

int gemmQ40TcV(int epi, const void *qs, const void *scales, uint32_t d, uint32_t n, const void *act, uint32_t actStride, uint32_t T,
               void *out, uint32_t outStride, int numSms, cudaStream_t stream, bool pdl, int variant) {
    const GemmPlan p = planGemmQ40Tc(epi, d, n, T, actStride, numSms, variant);
    if (p.rc) return p.rc;
    EncodeTiledFn enc = encodeTiled();
    if (!enc) return -2;
    GemmArgs a{};
    a.act = gHiddenAct;
    a.qs = (const uint32_t *)qs; a.scales = (const __half *)scales; a.d = d; a.n = n; a.T = T;
    a.out = out; a.outStride = outStride;
    a.stages = p.stages; a.rawStages = p.rawStages; a.bStages = p.bStages;

    CUtensorMap mapB, mapQ, mapS;
    if (!encode2d(enc, &mapB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, act, n, T, (uint64_t)actStride * 2, kGmBlockK, kGmTokTile, CU_TENSOR_MAP_SWIZZLE_128B))
        return -4;
    if (p.tma) {
        if (!encode2d(enc, &mapQ, CU_TENSOR_MAP_DATA_TYPE_UINT8, qs, n / 2, d, n / 2, 128, kGmBlockM, CU_TENSOR_MAP_SWIZZLE_128B)) return -7;
        if (!encode2d(enc, &mapS, CU_TENSOR_MAP_DATA_TYPE_UINT8, scales, n / 16, d, n / 16, 16, kGmBlockM, CU_TENSOR_MAP_SWIZZLE_NONE)) return -8;
    }
    a.splitK = p.splitK;
    if (p.splitK >= 2) {
        const size_t need = (size_t)p.splitK * T * d * sizeof(float);
        if (need > gSplitScratchBytes) {
            if (gSplitScratch) cudaFree(gSplitScratch);
            DL_CUDA_CHECK(cudaMalloc(&gSplitScratch, need));
            gSplitScratchBytes = need;
        }
        if (!gSplitCounters) {
            DL_CUDA_CHECK(cudaMalloc(&gSplitCounters, 4096 * sizeof(unsigned int)));
            DL_CUDA_CHECK(cudaMemset(gSplitCounters, 0, 4096 * sizeof(unsigned int)));
        }
        a.splitScratch = gSplitScratch; a.splitCounters = gSplitCounters;
        a.clusterSplit = p.clusterSplit;
    }
    const int grid = (int)p.grid;
    const CUtensorMap *pq = p.tma ? &mapQ : nullptr, *ps = p.tma ? &mapS : nullptr;
    switch (epi) {
        case GEPI_STORE_F32: return launchGemm<GEPI_STORE_F32>(mapB, pq, ps, a, grid, p.smemBytes, stream, pdl);
        case GEPI_RESIDUAL: return launchGemm<GEPI_RESIDUAL>(mapB, pq, ps, a, grid, p.smemBytes, stream, pdl);
        case GEPI_SWIGLU_BF16: return launchGemm<GEPI_SWIGLU_BF16>(mapB, pq, ps, a, grid, p.smemBytes, stream, pdl);
    }
    return -5;
}

// Grouped GEMM for mixture-of-experts prefill: nGroups stacked [grpRows][n] q40 matrices (the experts of one layer), activation rows
// sorted by expert. act: bf16 [rowsTotal][n]; grpCount / grpOffset: device arrays (moeSortKernel); maxTokens bounds the tokens of
// one group (the prompt chunk length: a token visits an expert at most once). Output rows follow the sorted order.
int gemmQ40TcGrouped(int epi, const void *qs, const void *scales, uint32_t nGroups, uint32_t grpRows, uint32_t n, const void *act,
                     uint32_t actStride, uint32_t rowsTotal, uint32_t maxTokens, const int *grpCount, const int *grpOffset, void *out,
                     uint32_t outStride, int numSms, cudaStream_t stream) {
    if (maxTokens == 0 || maxTokens > 256 || n % 256 || grpRows % 2 || (epi != GEPI_STORE_F32 && epi != GEPI_SWIGLU_BF16)) return 1;
    EncodeTiledFn enc = encodeTiled();
    if (!enc) return -2;
    GemmArgs a{};
    a.act = gHiddenAct;
    a.qs = (const uint32_t *)qs; a.scales = (const __half *)scales; a.d = nGroups * grpRows; a.n = n; a.T = maxTokens;
    a.out = out; a.outStride = outStride;
    a.grpCount = grpCount; a.grpOffset = grpOffset; a.grpRows = grpRows; a.grpTiles = (grpRows + kGmBlockM - 1) / kGmBlockM; a.nGroups = nGroups;
    a.splitK = 1;
    const size_t smemBytes = tmaGeometry(a);
    if (!smemBytes) return 1;
    CUtensorMap mapB, mapQ, mapS;
    if (!encode2d(enc, &mapB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, act, n, rowsTotal, (uint64_t)actStride * 2, kGmBlockK, kGmTokTile, CU_TENSOR_MAP_SWIZZLE_128B)) return -4;
    if (!encode2d(enc, &mapQ, CU_TENSOR_MAP_DATA_TYPE_UINT8, qs, n / 2, a.d, n / 2, 128, kGmBlockM, CU_TENSOR_MAP_SWIZZLE_128B)) return -7;
    if (!encode2d(enc, &mapS, CU_TENSOR_MAP_DATA_TYPE_UINT8, scales, n / 16, a.d, n / 16, 16, kGmBlockM, CU_TENSOR_MAP_SWIZZLE_NONE)) return -8;
    const uint32_t nItems = nGroups * a.grpTiles * ((maxTokens + kGmTokTile - 1) / kGmTokTile);
    const int grid = (int)(nItems < (uint32_t)numSms ? nItems : (uint32_t)numSms);
    switch (epi) {
        case GEPI_STORE_F32: return launchGemm<GEPI_STORE_F32>(mapB, &mapQ, &mapS, a, grid, smemBytes, stream, false);
        case GEPI_SWIGLU_BF16: return launchGemm<GEPI_SWIGLU_BF16>(mapB, &mapQ, &mapS, a, grid, smemBytes, stream, false);
    }
    return -5;
}

int gemmQ40Tc(int epi, const void *qs, const void *scales, uint32_t d, uint32_t n, const void *act, uint32_t actStride, uint32_t T,
              void *out, uint32_t outStride, int numSms, cudaStream_t stream, bool pdl) {
    return gemmQ40TcV(epi, qs, scales, d, n, act, actStride, T, out, outStride, numSms, stream, pdl, 0);
}

// ---- rmsnorm -> bf16 (activation operand producer) ------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsNormBf16Kernel(const float *__restrict__ x, uint32_t xStride, const float *__restrict__ w,
                                                         __nv_bfloat16 *__restrict__ y, uint32_t yStride, uint32_t n, float eps) {
    pdlLaunchDependents();
    pdlWait();
    __shared__ float red[8];
    const float4 *x4 = reinterpret_cast<const float4 *>(x + (size_t)blockIdx.x * xStride);
    float ss = 0.f;
    for (uint32_t i = threadIdx.x; i < n / 4; i += 256) {
        const float4 v = x4[i];
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warpSum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < 8; i++) tot += red[i];
    const float inv = rsqrtf(tot / (float)n + eps);
    __nv_bfloat162 *y2 = reinterpret_cast<__nv_bfloat162 *>(y + (size_t)blockIdx.x * yStride);
    for (uint32_t i = threadIdx.x; i < n / 4; i += 256) {
        const float4 v = x4[i];
        const float4 ww = w ? reinterpret_cast<const float4 *>(w)[i] : make_float4(1.f, 1.f, 1.f, 1.f);
        const float s = w ? inv : 1.f;
        y2[2 * i] = __floats2bfloat162_rn(ww.x * (v.x * s), ww.y * (v.y * s));
        y2[2 * i + 1] = __floats2bfloat162_rn(ww.z * (v.z * s), ww.w * (v.w * s));
    }
}

int launchRmsNormBf16(const float *x, uint32_t xStride, const float *w, void *y, uint32_t yStride, uint32_t n, float eps, uint32_t T,
                      cudaStream_t stream, bool pdl) {
    DL_CUDA_CHECK(launchPdl(rmsNormBf16Kernel, dim3(T), dim3(256), 0, stream, pdl, x, xStride, w, (__nv_bfloat16 *)y, yStride, n, eps));
    return 0;
}

}  // namespace dl

// Stand-alone entry point (tests, tools): the gate activation of GEPI_SWIGLU_BF16 is passed explicitly (0 = SiLU, 1 = GELU).
DL_EXPORT int dl_gemm_q40_tc(int epi, const void *qs, const void *scales, uint32_t d, uint32_t n, const void *act, uint32_t actStride,
                             uint32_t T, void *out, uint32_t outStride, int numSms, uint32_t hiddenAct, cudaStream_t stream, int pdl, int variant) {
    const dl::HiddenActScope a(hiddenAct);
    return dl::gemmQ40TcV(epi, qs, scales, d, n, act, actStride, T, out, outStride, numSms, stream, pdl != 0, variant);
}

// What dl_gemm_q40_tc would run for these arguments (and the current DL_GEMM_* switches), without launching or allocating:
// out[8] = {rc, kernel (1 register-prefetch, 2 TMA-staged), splitK, cluster reduce (0/1), grid, A stages, raw stages, B stages}.
DL_EXPORT int dl_gemm_q40_tc_plan(int epi, uint32_t d, uint32_t n, uint32_t T, uint32_t actStride, int numSms, int variant, int *out) {
    const dl::GemmPlan p = dl::planGemmQ40Tc(epi, d, n, T, actStride, numSms, variant);
    const int v[8] = {p.rc, p.tma ? 2 : 1, (int)p.splitK, (int)p.clusterSplit, (int)p.grid, (int)p.stages, (int)p.rawStages, (int)p.bStages};
    for (int i = 0; i < 8; i++) out[i] = p.rc ? (i == 0 ? p.rc : 0) : v[i];
    return p.rc;
}

// Grouped mode for the unit tests (tests/test_gpu_moe.py): gemmQ40TcGrouped with caller-provided device arrays grpCount /
// grpOffset [nGroups] and the gate activation of GEPI_SWIGLU_BF16 passed explicitly (0 = SiLU, 1 = GELU).
DL_EXPORT int dl_gemm_q40_tc_grouped(int epi, const void *qs, const void *scales, uint32_t nGroups, uint32_t grpRows, uint32_t n, const void *act,
                                     uint32_t actStride, uint32_t rowsTotal, uint32_t maxTokens, const int *grpCount, const int *grpOffset,
                                     void *out, uint32_t outStride, int numSms, uint32_t hiddenAct, cudaStream_t stream) {
    const dl::HiddenActScope a(hiddenAct);
    return dl::gemmQ40TcGrouped(epi, qs, scales, nGroups, grpRows, n, act, actStride, rowsTotal, maxTokens, grpCount, grpOffset, out,
                                outStride, numSms, stream);
}

DL_EXPORT int dl_rmsnorm_bf16(const float *x, uint32_t xStride, const float *w, void *y, uint32_t yStride, uint32_t n, float eps,
                              uint32_t T, cudaStream_t stream) {
    return dl::launchRmsNormBf16(x, xStride, w, y, yStride, n, eps, T, stream);
}
