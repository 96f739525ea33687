// Prompt-chunk (prefill) attention on the Hopper tensor cores: S = Q.K^T and O = P.V are wgmma.mma_async instructions with the
// accumulators in registers; K and V tiles stream from the bf16 head-major KV cache through TMA tensor maps.
// The maps are 3-D, {headDim, p0 + T, nKvHeads}, so TMA fills the rows of a tile at or past p0 + T with zeros: the kernel reads only
// rows [0, p0 + T) of its own head, never a later (not yet written, or a previous request's) row or the next head's rows. Those rows
// are masked to P = 0, but 0 * NaN is NaN on the tensor core as anywhere else.
// A paged slot (PAGED kernels) reads its rows through its page table instead, and zeroes the rows past p0 + T itself.
//
// Work item (one CTA) = one KV head x one query tile. The `kvMul` query heads that share the KV head (GQA) are packed on the
// MMA M dimension: a tile holds tq = 128 / kvMul consecutive prompt tokens x kvMul heads = up to 128 query rows, so every K / V
// tile fetched from the cache is used by all heads of the group. KV is walked in tiles of 128 positions, causal inside the chunk
// (row of token t sees positions <= p0 + t). Two passes over the KV tiles keep the kernel free of accumulator rescaling:
//   pass 1: S tiles -> per-row running maximum m and normaliser l
//   pass 2: S tiles again -> P = exp2(S - m) as bf16 registers (the A operand of the next wgmma) -> O += P.V
// Warp roles: 0 = TMA producer; warps 4..7 and 8..11 = two consumer warpgroups, each owning 64 query rows of the tile (wgmma M = 64).
// A q80 cache (the Q8 variant) has no TMA path: warps 0..3 read the int8 rows and their scales, widen them to bf16 and store them in
// the same swizzled layout the TMA would have produced; everything after the full barrier is the same kernel.
// Each 128-position KV tile is processed as two halves of 64 positions (S half = 32 registers a thread).
//
// Replaces (reference): OP_MULTIHEAD_ATT over a prompt chunk, multiheadAtt_F32 + softmax_F32 per (head, batch row)
// (src/nn/nn-cpu-ops.cpp:753-788,1260-1286) and the round-1 fallback that ran the decode kernel once per (head, token).
#include <cuda.h>

#include <type_traits>

#include "kernels.h"
#include "wgmma.cuh"

namespace dl {
namespace {

constexpr int kApThreads = 384;
constexpr uint32_t kApAtomBytes = 16384;   // one [128 rows x 64 bf16] SWIZZLE_128B atom column
constexpr uint32_t kApConsumerWarps = 8;

__device__ __forceinline__ uint32_t apAddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void apBarInit(uint64_t *b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(apAddr(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void apBarExpectTx(uint64_t *b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(apAddr(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void apBarArrive(uint64_t *b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(apAddr(b)) : "memory"); }
__device__ __forceinline__ void apBarWait(uint64_t *b, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nAP_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra AP_DONE;\nbra AP_WAIT;\nAP_DONE:\n}\n" ::"r"(apAddr(b)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void apTmaLoad3d(void *dst, const CUtensorMap *map, uint32_t c0, uint32_t c1, uint32_t c2, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(apAddr(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(apAddr(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ uint32_t apPack(float lo, float hi) {
    __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&b);
}

struct AttnPrefillKArgs {
    const float *qkv;           // [T][qkvStride] f32; the q rows are already normalised + rotated (ropeKvKernel)
    uint32_t qkvStride;
    uint32_t T, p0;             // the chunk holds the tokens at positions p0 .. p0 + T - 1
    uint32_t nHeads, nKvHeads, seqLen;
    uint32_t kvMul, tq, nQTiles;   // query heads per KV head, tokens per query tile, query tiles per KV head
    __nv_bfloat16 *out;         // [T][outStride]: token-major, head h at columns h * HD
    uint32_t outStride;
    float scaleLog2;            // log2(e) / sqrt(headDim), folded into q
    const int8_t *kQ8, *vQ8;    // q80 cache (Q8 kernels): value planes and scale planes [nKvHeads][seqLen][HD / 32]
    const __half *kScale, *vScale;
};

// The arguments of the PAGED kernels (derived, so that the others keep their argument layout and their code).
struct PagedPrefillKArgs : AttnPrefillKArgs {
    const __nv_bfloat16 *vBf16; // bf16: the V plane (the tile past the chunk's last row is copied, not loaded by TMA)
    const int32_t *pageTable;   // the slot's page table (logical row r at physical row table[r / 64] * 64 + r % 64)
};
template <bool PAGED> using PrefillKArgs = typename std::conditional<PAGED, PagedPrefillKArgs, AttnPrefillKArgs>::type;
template <typename A>
__device__ __forceinline__ const int32_t *pagesOf(const A &a) {
    if constexpr (std::is_same<A, PagedPrefillKArgs>::value) return a.pageTable;
    else return nullptr;
}

// Q8: one 128-position K or V tile of a q80 cache, widened to bf16 by the 128 threads of warps 0..3 into the SWIZZLE_128B layout
// ([NA][128 rows][128 B], 16-byte chunk c of row r at ((c ^ (r & 7)) << 4)). Rows at or past `rowEnd` (not yet written) are zero.
// PAGED: logical row pos0 + r is read from its page.
template <int HD, bool PAGED>
__device__ __forceinline__ void apWidenTile(uint8_t *dst, const int8_t *q, const __half *sc, uint32_t kvRow0, uint32_t pos0, uint32_t rowEnd,
                                            const int32_t *table) {
    constexpr uint32_t CPR = HD / 8;   // 16-byte bf16 chunks per row
    for (uint32_t u = threadIdx.x; u < 128 * CPR; u += 128) {
        const uint32_t r = u / CPR, cc = u % CPR;
        uint4 packed = make_uint4(0u, 0u, 0u, 0u);
        if (pos0 + r < rowEnd) {
            size_t e;
            if constexpr (PAGED) e = (size_t)(kvRow0 + pagedRow(table, pos0 + r)) * HD + cc * 8;
            else e = (size_t)(kvRow0 + pos0 + r) * HD + cc * 8;
            const float d = __half2float(sc[e / 32]);
            const uint2 w = *reinterpret_cast<const uint2 *>(q + e);
            packed = make_uint4(apPack(q8ToFloat(w.x, 0) * d, q8ToFloat(w.x, 1) * d), apPack(q8ToFloat(w.x, 2) * d, q8ToFloat(w.x, 3) * d),
                                apPack(q8ToFloat(w.y, 0) * d, q8ToFloat(w.y, 1) * d), apPack(q8ToFloat(w.y, 2) * d, q8ToFloat(w.y, 3) * d));
        }
        *reinterpret_cast<uint4 *>(dst + (cc >> 3) * kApAtomBytes + r * 128 + (((cc & 7) ^ (r & 7)) << 4)) = packed;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
    __syncwarp();
}

// PAGED bf16: the V tile that holds rows at or past `rowEnd`, copied by the 32 lanes of warp 0 into the SWIZZLE_128B layout. Those rows
// of a page may hold anything (another request's rows, or NaN); they get P = 0, and 0 * NaN would still be NaN, so they are zeroed.
template <int HD>
__device__ __forceinline__ void apCopyTailTile(uint8_t *dst, const __nv_bfloat16 *plane, uint32_t kvRow0, uint32_t pos0, uint32_t rowEnd,
                                               const int32_t *table) {
    constexpr uint32_t CPR = HD / 8;
    for (uint32_t u = threadIdx.x & 31; u < 128 * CPR; u += 32) {
        const uint32_t r = u / CPR, cc = u % CPR;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (pos0 + r < rowEnd) v = *reinterpret_cast<const uint4 *>(plane + (size_t)(kvRow0 + pagedRow(table, pos0 + r)) * HD + cc * 8);
        *reinterpret_cast<uint4 *>(dst + (cc >> 3) * kApAtomBytes + r * 128 + (((cc & 7) ^ (r & 7)) << 4)) = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
}

// PAGED: the slot's rows are read through its page table (AttnPrefillKArgs::pageTable) from a map over the whole layer plane: a
// 128-position K tile is two 64-row TMA boxes at the pages' physical rows, and the last V tile of a query tile comes through
// apCopyTailTile. The tiles, and so the arithmetic, are those of a contiguous cache.
template <int HD, bool Q8, bool PAGED>
__global__ void __launch_bounds__(kApThreads, 1) attnPrefillTcKernel(const __grid_constant__ CUtensorMap tmapK,
                                                                     const __grid_constant__ CUtensorMap tmapV, PrefillKArgs<PAGED> a) {
    constexpr uint32_t NA = HD / 64;                    // 64-wide atom columns along headDim
    constexpr uint32_t kTileBytes = NA * kApAtomBytes;  // one K or V tile: 128 positions x HD
    extern __shared__ __align__(1024) uint8_t apSmemRaw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(apSmemRaw) + 1023) & ~(uintptr_t)1023);
    uint8_t *Qs = smem;                                  // [NA][128 rows][128 B]
    uint8_t *Ks = Qs + kTileBytes;                       // [2][NA][128][128 B]
    uint8_t *Vs = Ks + 2 * kTileBytes;                   // [2][NA][128][128 B]
    uint64_t *bars = reinterpret_cast<uint64_t *>(Vs + 2 * kTileBytes);
    uint64_t *kFull = bars, *kEmpty = bars + 2, *vFull = bars + 4, *vEmpty = bars + 6;

    // warp index via shuffle = warp-uniform for the compiler: the role branches become uniform control flow
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const uint32_t item = blockIdx.x;
    const uint32_t kvh = item / a.nQTiles, qt = item - kvh * a.nQTiles;
    const uint32_t t0 = qt * a.tq;
    const uint32_t tqValid = min(a.tq, a.T - t0);
    const uint32_t rowsValid = tqValid * a.kvMul;
    const uint32_t nKv = (a.p0 + t0 + tqValid + 127) / 128;      // KV tiles this query tile can see
    const uint32_t kvRow0 = kvh * a.seqLen;

    pdlLaunchDependents();
    if (tid == 0) {
        const uint32_t fills = Q8 ? 4 : 1;   // Q8: the lane 0 of each of warps 0..3 arrives once its rows are stored
        for (int i = 0; i < 2; i++) {
            apBarInit(&kFull[i], fills); apBarInit(&kEmpty[i], kApConsumerWarps);
            apBarInit(&vFull[i], fills); apBarInit(&vEmpty[i], kApConsumerWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdlWait();   // q rows and the new K/V rows come from the rope kernel before this one

    if (Q8 && warp < 4) {
        // ================================ q80 producer: warps 0..3 ================================
        const uint32_t rowEnd = a.p0 + a.T;   // rows [0, p0 + T) of the head are in the cache
        uint32_t itK = 0;
        for (uint32_t pass = 0; pass < 2; pass++) {
            for (uint32_t j = 0; j < nKv; j++, itK++) {
                const uint32_t st = itK & 1, ph = (itK >> 1) & 1;
                apBarWait(&kEmpty[st], ph ^ 1);
                apWidenTile<HD, PAGED>(Ks + st * kTileBytes, a.kQ8, a.kScale, kvRow0, j * 128, rowEnd, pagesOf(a));
                if (lane == 0) apBarArrive(&kFull[st]);
                if (pass == 1) {
                    const uint32_t vs = j & 1, vph = (j >> 1) & 1;
                    apBarWait(&vEmpty[vs], vph ^ 1);
                    apWidenTile<HD, PAGED>(Vs + vs * kTileBytes, a.vQ8, a.vScale, kvRow0, j * 128, rowEnd, pagesOf(a));
                    if (lane == 0) apBarArrive(&vFull[vs]);
                }
            }
        }
    } else if (!Q8 && PAGED && warp == 0) {
        // ============================ TMA producer, paged: warp 0 ============================
        if constexpr (PAGED) {
        const uint32_t rowEnd = a.p0 + a.T;
        uint32_t itK = 0;
        for (uint32_t pass = 0; pass < 2; pass++) {
            for (uint32_t j = 0; j < nKv; j++, itK++) {
                const uint32_t st = itK & 1, ph = (itK >> 1) & 1;
                apBarWait(&kEmpty[st], ph ^ 1);
                if (lane == 0) {
                    // page 2j holds a row below rowEnd; a page 2j + 1 past it is loaded as page 2j again (masked like any row past rowEnd)
                    const uint32_t r0 = (uint32_t)__ldg(a.pageTable + 2 * j) * 64;
                    const uint32_t r1 = j * 128 + 64 < rowEnd ? (uint32_t)__ldg(a.pageTable + 2 * j + 1) * 64 : r0;
                    apBarExpectTx(&kFull[st], kTileBytes);
                    for (uint32_t c = 0; c < NA; c++) {
                        apTmaLoad3d(Ks + st * kTileBytes + c * kApAtomBytes, &tmapK, c * 64, r0, kvh, &kFull[st]);
                        apTmaLoad3d(Ks + st * kTileBytes + c * kApAtomBytes + 8192, &tmapK, c * 64, r1, kvh, &kFull[st]);
                    }
                }
                if (pass == 1) {
                    const uint32_t vs = j & 1, vph = (j >> 1) & 1;
                    apBarWait(&vEmpty[vs], vph ^ 1);
                    if (j * 128 + 128 > rowEnd) {
                        apCopyTailTile<HD>(Vs + vs * kTileBytes, a.vBf16, kvRow0, j * 128, rowEnd, a.pageTable);
                        if (lane == 0) apBarArrive(&vFull[vs]);
                    } else if (lane == 0) {
                        const uint32_t r0 = (uint32_t)__ldg(a.pageTable + 2 * j) * 64, r1 = (uint32_t)__ldg(a.pageTable + 2 * j + 1) * 64;
                        apBarExpectTx(&vFull[vs], kTileBytes);
                        for (uint32_t c = 0; c < NA; c++) {
                            apTmaLoad3d(Vs + vs * kTileBytes + c * kApAtomBytes, &tmapV, c * 64, r0, kvh, &vFull[vs]);
                            apTmaLoad3d(Vs + vs * kTileBytes + c * kApAtomBytes + 8192, &tmapV, c * 64, r1, kvh, &vFull[vs]);
                        }
                    }
                }
            }
        }
        }
    } else if (!Q8 && !PAGED && warp == 0) {
        // ================================ TMA producer ================================
        // expect_tx counts the whole box: TMA delivers the zero-filled rows past p0 + T like the loaded ones
        if (lane == 0) {
            uint32_t itK = 0;
            for (uint32_t pass = 0; pass < 2; pass++) {
                for (uint32_t j = 0; j < nKv; j++, itK++) {
                    const uint32_t st = itK & 1, ph = (itK >> 1) & 1;
                    apBarWait(&kEmpty[st], ph ^ 1);
                    apBarExpectTx(&kFull[st], kTileBytes);
                    for (uint32_t c = 0; c < NA; c++) apTmaLoad3d(Ks + st * kTileBytes + c * kApAtomBytes, &tmapK, c * 64, j * 128, kvh, &kFull[st]);
                    if (pass == 1) {
                        const uint32_t vs = j & 1, vph = (j >> 1) & 1;
                        apBarWait(&vEmpty[vs], vph ^ 1);
                        apBarExpectTx(&vFull[vs], kTileBytes);
                        for (uint32_t c = 0; c < NA; c++) apTmaLoad3d(Vs + vs * kTileBytes + c * kApAtomBytes, &tmapV, c * 64, j * 128, kvh, &vFull[vs]);
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // ============================ consumer warpgroup g: query rows [64g, 64g + 64) ============================
        const uint32_t g = (uint32_t)(warp - 4) >> 2, qw = (uint32_t)(warp - 4) & 3;
        // ---- Q rows of this warpgroup: f32 -> scaled bf16, canonical K-major SWIZZLE_128B layout ----
        {
            constexpr uint32_t CPR = HD / 8;           // 16-byte chunks (8 elements) per row
            constexpr uint32_t RPI = 32 / CPR;         // rows per warp iteration
            const uint32_t cc = lane % CPR;
            for (uint32_t r0 = 64 * g + 16 * qw; r0 < 64 * g + 16 * qw + 16; r0 += RPI) {
                const uint32_t r = r0 + lane / CPR;
                uint4 packed = make_uint4(0u, 0u, 0u, 0u);
                if (r < rowsValid) {
                    const uint32_t ti = r / a.kvMul, hi = r - ti * a.kvMul;
                    const float4 *src = reinterpret_cast<const float4 *>(a.qkv + (size_t)(t0 + ti) * a.qkvStride + (size_t)(kvh * a.kvMul + hi) * HD + cc * 8);
                    const float4 v0 = __ldg(src), v1 = __ldg(src + 1);
                    const float s = a.scaleLog2;
                    packed = make_uint4(apPack(v0.x * s, v0.y * s), apPack(v0.z * s, v0.w * s), apPack(v1.x * s, v1.y * s), apPack(v1.z * s, v1.w * s));
                }
                *reinterpret_cast<uint4 *>(Qs + (cc >> 3) * kApAtomBytes + r * 128 + (((cc & 7) ^ (r & 7)) << 4)) = packed;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
            wgBarrier(1 + g);
        }
        // this thread's two accumulator rows (fragment rows lane / 4 and lane / 4 + 8 of the warp's 16)
        bool rowOk[2];
        uint32_t rowPos[2];   // last visible position of the row
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t row = 64 * g + 16 * qw + (lane >> 2) + 8 * h;
            rowOk[h] = row < rowsValid;
            rowPos[h] = a.p0 + t0 + row / a.kvMul;
        }
        const uint32_t qAddr = apAddr(Qs) + g * 8192;          // rows 64g.. start 64 x 128 B into every atom
        const uint32_t colBase = 2 * (lane & 3);
        // S half-tile [64 rows x 64 positions] = Q . K^T, K rows [half * 64, half * 64 + 64) of the stage
        auto computeS = [&](float (&s)[32], uint32_t kAddr) {
            wgFence();
#pragma unroll
            for (uint32_t c = 0; c < NA; c++)
#pragma unroll
                for (uint32_t k = 0; k < 4; k++)
                    wgmmaSS<0>(s, wgDesc(qAddr + c * kApAtomBytes) + 2 * k, wgDesc(kAddr + c * kApAtomBytes) + 2 * k, (c | k) != 0 ? 1u : 0u);
            wgCommit();
            wgWait<0>();
            wgFenceAcc(s);
        };
        // causal mask in place (masked -> -inf); fragment element 4i + 2h + e = (row h, position pos0 + 8i + colBase + e)
        auto maskS = [&](float (&s)[32], uint32_t pos0) {
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const bool vis = rowOk[h] && pos0 + 8 * i + colBase + e <= rowPos[h];
                        if (!vis) s[4 * i + 2 * h + e] = -INFINITY;
                    }
        };
        float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
        uint32_t itK = 0;
        // ---- pass 1: row maximum and normaliser ----
        for (uint32_t j = 0; j < nKv; j++, itK++) {
            const uint32_t st = itK & 1, ph = (itK >> 1) & 1;
            apBarWait(&kFull[st], ph);
#pragma unroll 1
            for (uint32_t half = 0; half < 2; half++) {
                float s[32];
                computeS(s, apAddr(Ks + st * kTileBytes) + half * 8192);
                maskS(s, j * 128 + half * 64);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    float cm = -INFINITY;
#pragma unroll
                    for (int i = 0; i < 8; i++) cm = fmaxf(cm, fmaxf(s[4 * i + 2 * h], s[4 * i + 2 * h + 1]));
                    cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
                    cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));   // the 4 lanes of a row
                    const float mNew = fmaxf(m[h], cm);
                    float acc = 0.f;
                    if (mNew > -INFINITY) {
#pragma unroll
                        for (int i = 0; i < 8; i++) acc += exp2f(s[4 * i + 2 * h] - mNew) + exp2f(s[4 * i + 2 * h + 1] - mNew);
                    }
                    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
                    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
                    if (mNew > -INFINITY) {
                        l[h] = l[h] * exp2f(m[h] - mNew) + acc;
                        m[h] = mNew;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) apBarArrive(&kEmpty[st]);
        }
        // ---- pass 2: P = exp2(S - m) -> O += P.V ----
        const float mP[2] = {m[0] > -INFINITY ? m[0] : 0.f, m[1] > -INFINITY ? m[1] : 0.f};   // rows without a visible position: P = 0
        float o[NA][32];
        for (uint32_t j = 0; j < nKv; j++, itK++) {
            const uint32_t st = itK & 1, ph = (itK >> 1) & 1, vs = j & 1, vph = (j >> 1) & 1;
            apBarWait(&kFull[st], ph);
            apBarWait(&vFull[vs], vph);
#pragma unroll 1
            for (uint32_t half = 0; half < 2; half++) {
                float s[32];
                computeS(s, apAddr(Ks + st * kTileBytes) + half * 8192);
                maskS(s, j * 128 + half * 64);
                uint32_t pa[4][4];   // A fragments of 4 k-steps of 16 positions
#pragma unroll
                for (int kk = 0; kk < 4; kk++)
#pragma unroll
                    for (int x = 0; x < 4; x++) {
                        const int i = 2 * kk + (x >> 1), h = x & 1;   // a0: (i = 2kk, row), a1: (2kk, row + 8), a2: (2kk + 1, row), a3: (2kk + 1, row + 8)
                        pa[kk][x] = apPack(exp2f(s[4 * i + 2 * h] - mP[h]), exp2f(s[4 * i + 2 * h + 1] - mP[h]));
                    }
                wgFence();
#pragma unroll
                for (int kk = 0; kk < 4; kk++)
#pragma unroll
                    for (uint32_t n = 0; n < NA; n++) {
                        const uint32_t vAddr = apAddr(Vs + vs * kTileBytes + n * kApAtomBytes) + (half * 64 + kk * 16) * 128;
                        wgmmaRS(o[n], pa[kk], wgDesc(vAddr, kApAtomBytes), (j | half | kk) != 0 ? 1u : 0u);
                    }
                wgCommit();
                wgWait<0>();
#pragma unroll
                for (uint32_t n = 0; n < NA; n++) wgFenceAcc(o[n]);
            }
            __syncwarp();
            if (lane == 0) {
                apBarArrive(&kEmpty[st]);
                apBarArrive(&vEmpty[vs]);
            }
        }
        // ---- epilogue: O / l -> bf16 ----
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!rowOk[h]) continue;
            const uint32_t row = 64 * g + 16 * qw + (lane >> 2) + 8 * h;
            const uint32_t ti = row / a.kvMul, hi = row - ti * a.kvMul;
            const float invL = l[h] > 0.f ? 1.f / l[h] : 0.f;
            __nv_bfloat16 *orow = a.out + (size_t)(t0 + ti) * a.outStride + (size_t)(kvh * a.kvMul + hi) * HD;
#pragma unroll
            for (uint32_t n = 0; n < NA; n++)
#pragma unroll
                for (int i = 0; i < 8; i++)
                    *reinterpret_cast<uint32_t *>(orow + n * 64 + 8 * i + colBase) = apPack(o[n][4 * i + 2 * h] * invL, o[n][4 * i + 2 * h + 1] * invL);
        }
    }
}

typedef CUresult (*ApEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                               const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

ApEncodeFn apEncode() {
    static ApEncodeFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<ApEncodeFn>(p);
    }
    return fn;
}

// Rows [0, rows) of every head of a [nKvHeads][seqLen][hd] bf16 cache; a box is 64 columns x boxRows rows of one head.
bool apCacheMap(CUtensorMap *map, const void *cache, uint32_t hd, uint32_t rows, uint32_t nKvHeads, uint32_t seqLen, uint32_t boxRows = 128) {
    ApEncodeFn enc = apEncode();
    if (!enc) return false;
    const cuuint64_t dims[3] = {hd, rows, nKvHeads};
    const cuuint64_t strides[2] = {(cuuint64_t)hd * 2, (cuuint64_t)hd * 2 * seqLen};
    const cuuint32_t box[3] = {64, boxRows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(cache), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int HD, bool Q8, bool PAGED>
int apLaunch(const CUtensorMap &mk, const CUtensorMap &mv, const PrefillKArgs<PAGED> &k, uint32_t grid, cudaStream_t stream, bool pdl) {
    constexpr size_t smemBytes = (size_t)(HD / 64) * kApAtomBytes * 5 + 256 + 1024;
    static bool configured = false;
    if (!configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(attnPrefillTcKernel<HD, Q8, PAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
        configured = true;
    }
    DL_CUDA_CHECK(launchPdl(attnPrefillTcKernel<HD, Q8, PAGED>, dim3(grid), dim3(kApThreads), smemBytes, stream, pdl, mk, mv, k));
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

// A paged slot's chunk: q80 widened through the table; bf16 over maps of the whole layer plane in 64-row boxes (one page each).
int launchPaged(const AttnPrefillArgs &a, const AttnPrefillKArgs &base, uint32_t grid, cudaStream_t stream, bool pdl) {
    PagedPrefillKArgs k{};
    static_cast<AttnPrefillKArgs &>(k) = base;
    k.pageTable = a.pageTable;
    if (a.kScale) {
        CUtensorMap none{};
        k.kQ8 = (const int8_t *)a.kCache; k.vQ8 = (const int8_t *)a.vCache; k.kScale = a.kScale; k.vScale = a.vScale;
        return a.headDim == 128 ? apLaunch<128, true, true>(none, none, k, grid, stream, pdl) : apLaunch<64, true, true>(none, none, k, grid, stream, pdl);
    }
    CUtensorMap mk, mv;
    if (!apCacheMap(&mk, a.kCache, a.headDim, a.seqLen, a.nKvHeads, a.seqLen, 64) || !apCacheMap(&mv, a.vCache, a.headDim, a.seqLen, a.nKvHeads, a.seqLen, 64))
        return -2;
    k.vBf16 = (const __nv_bfloat16 *)a.vCache;
    return a.headDim == 128 ? apLaunch<128, false, true>(mk, mv, k, grid, stream, pdl) : apLaunch<64, false, true>(mk, mv, k, grid, stream, pdl);
}

}  // namespace

// Returns 1 when the shape is not covered (caller falls back to the per-token kernel).
int launchAttnPrefillTc(const AttnPrefillArgs &a, cudaStream_t stream, bool pdl) {
    if (a.headDim != 64 && a.headDim != 128) return 1;
    if (a.nKvHeads == 0 || a.nHeads % a.nKvHeads) return 1;
    const uint32_t kvMul = a.nHeads / a.nKvHeads;
    if (kvMul > 128 || a.T == 0) return 1;
    if (a.p0 + a.T > a.seqLen) return -1;
    AttnPrefillKArgs k{};
    k.qkv = a.qkv; k.qkvStride = a.qkvStride; k.T = a.T; k.p0 = a.p0; k.nHeads = a.nHeads; k.nKvHeads = a.nKvHeads; k.seqLen = a.seqLen;
    k.kvMul = kvMul; k.tq = 128 / kvMul; k.nQTiles = (a.T + k.tq - 1) / k.tq;
    k.out = a.out; k.outStride = a.outStride;
    k.scaleLog2 = 1.4426950408889634f / sqrtf((float)a.headDim);
    const uint32_t grid = a.nKvHeads * k.nQTiles;
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    if (a.pageTable) return launchPaged(a, k, grid, stream, pdl);
    if (a.kScale) {   // q80: widened by the kernel itself, no tensor maps
        CUtensorMap none{};
        k.kQ8 = (const int8_t *)a.kCache; k.vQ8 = (const int8_t *)a.vCache; k.kScale = a.kScale; k.vScale = a.vScale;
        return a.headDim == 128 ? apLaunch<128, true, false>(none, none, k, grid, stream, pdl) : apLaunch<64, true, false>(none, none, k, grid, stream, pdl);
    }
    CUtensorMap mk, mv;
    const uint32_t rows = a.p0 + a.T;   // rows of each head this chunk may read; TMA zero-fills the rest of the last tile
    if (!apCacheMap(&mk, a.kCache, a.headDim, rows, a.nKvHeads, a.seqLen) || !apCacheMap(&mv, a.vCache, a.headDim, rows, a.nKvHeads, a.seqLen))
        return -2;
    return a.headDim == 128 ? apLaunch<128, false, false>(mk, mv, k, grid, stream, pdl) : apLaunch<64, false, false>(mk, mv, k, grid, stream, pdl);
}

}  // namespace dl

// Stand-alone entry point for the unit test (tests/test_gpu_attn_prefill.py): q rows are taken as given (no rope).
DL_EXPORT int dl_attn_prefill_tc(const float *qkv, uint32_t qkvStride, uint32_t T, uint32_t p0, uint32_t nHeads, uint32_t nKvHeads,
                                 uint32_t headDim, uint32_t seqLen, const void *kCache, const void *vCache, void *out, uint32_t outStride,
                                 cudaStream_t stream) {
    dl::AttnPrefillArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.T = T; a.p0 = p0; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = kCache; a.vCache = vCache; a.out = (__nv_bfloat16 *)out; a.outStride = outStride;
    return dl::launchAttnPrefillTc(a, stream);
}

// The same over a q80 cache: int8 value planes kCache / vCache, f16 scale planes kScale / vScale [nKvHeads][seqLen][headDim / 32].
DL_EXPORT int dl_attn_prefill_tc_q80(const float *qkv, uint32_t qkvStride, uint32_t T, uint32_t p0, uint32_t nHeads, uint32_t nKvHeads,
                                     uint32_t headDim, uint32_t seqLen, const void *kCache, const void *vCache, const void *kScale,
                                     const void *vScale, void *out, uint32_t outStride, cudaStream_t stream) {
    dl::AttnPrefillArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.T = T; a.p0 = p0; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = kCache; a.vCache = vCache; a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale;
    a.out = (__nv_bfloat16 *)out; a.outStride = outStride;
    return dl::launchAttnPrefillTc(a, stream);
}

// Tensor-core prefill attention of one paged slot's chunk (tests/test_gpu_paged_slots.py): kCache / vCache are whole layer planes of
// seqLen rows per KV head (seqLen a multiple of 64), pageTable (device int32) maps the slot's logical page i to physical page
// pageTable[i]; kScale / vScale null: bf16 planes, else q80 scale planes.
DL_EXPORT int dl_attn_prefill_tc_paged(const float *qkv, uint32_t qkvStride, uint32_t T, uint32_t p0, uint32_t nHeads, uint32_t nKvHeads,
                                       uint32_t headDim, uint32_t seqLen, const void *kCache, const void *vCache, const void *kScale,
                                       const void *vScale, const int32_t *pageTable, void *out, uint32_t outStride, cudaStream_t stream) {
    dl::AttnPrefillArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.T = T; a.p0 = p0; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = kCache; a.vCache = vCache; a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale; a.pageTable = pageTable;
    a.out = (__nv_bfloat16 *)out; a.outStride = outStride;
    return dl::launchAttnPrefillTc(a, stream);
}
