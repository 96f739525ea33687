// TMA-fed decode GEMV: y[t][d] = W_q40[d][n] · q80(x[t][n]), 1..8 tokens, fused prologue/epilogue.
//
// Same contract as gemv_q40.cu (which stays as the fallback for shapes the bulk-copy alignment rules reject), but
// the weight stream is moved by the TMA unit instead of by per-thread loads:
//   * warp 16 (one elected lane) is the producer: it cuts the CTA's contiguous row tile into stages of ~16-32 KB
//     and issues `cp.async.bulk` (global -> shared, mbarrier complete_tx) for nibbles and scales; a ring of up to
//     ~190 KB per SM is in flight, none of it costing registers;
//   * the ring is filled *before* griddepcontrol.wait, i.e. while the previous kernel of the layer is still
//     running (PDL) — weights are constants, only the activations depend on the predecessor;
//   * warps 0-15 consume: per step a warp takes 4 rows x 32 quant blocks from shared memory, the activation block
//     of each lane is read once and reused for the 4 rows (dp4a), 4 partial sums are reduced with a 6-shuffle
//     transposing butterfly, per-(row,segment) partials are summed in fixed order (deterministic);
//   * full/empty mbarrier pairs recycle stages when the tile is larger than the ring (w13, logits).
#include "gemv_common.cuh"

namespace dl {

struct TmaGemvGeom {
    uint32_t stageRows, nStages, stageBytes, maxTileRows;
};

// NB == 1 (decode) is compiled for two resident CTAs per SM: while kernel N computes, the CTAs of kernel N+1 are already
// on the SM (PDL) with their ring filling, so consecutive kernels of a layer overlap load and compute.
template <int PRO, int EPI, int NB>
__global__ void __launch_bounds__(kTmaThreads, (NB == 1 ? 2 : 1)) gemvQ40TmaKernel(GemvArgs a, TmaGemvGeom geo) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nblk = a.n / 32;
    const uint32_t nseg = (nblk + 31) / 32;
    const uint32_t rowQsBytes = nblk * 16, rowScBytes = nblk * 2;

    // ---- tile (pair aligned, like the fallback kernel); MoE launches carry one tile grid per routing slot ----
    const bool moe = a.moeCtasPerSlot != 0;
    const uint32_t nTiles = moe ? a.moeCtasPerSlot : gridDim.x;
    const uint32_t tileIdx = moe ? blockIdx.x % a.moeCtasPerSlot : blockIdx.x;
    const uint32_t slot = moe ? blockIdx.x / a.moeCtasPerSlot : 0;
    const uint32_t nPairs = a.d / 2;
    const uint32_t pairBegin = (uint32_t)(((uint64_t)tileIdx * nPairs) / nTiles);
    const uint32_t pairEnd = (uint32_t)(((uint64_t)(tileIdx + 1) * nPairs) / nTiles);
    const uint32_t rowBase = pairBegin * 2;
    const uint32_t tileRows = (pairEnd - pairBegin) * 2;
    const uint32_t SR = geo.stageRows;
    const uint32_t nFills = (tileRows + SR - 1) / SR;

    // ---- shared memory carve-up: [ring stages][planes][dx][dx8][partial][red][barriers] ----
    uint8_t *ring = smem;
    uint4 *planeA = reinterpret_cast<uint4 *>(ring + (size_t)geo.nStages * geo.stageBytes);
    uint4 *planeB = planeA + (size_t)NB * nblk;
    float *dxs = reinterpret_cast<float *>(planeB + (size_t)NB * nblk);
    float *dx8 = dxs + (size_t)NB * nblk;
    float *partial = dx8 + (size_t)NB * nblk;                               // [maxTileRows(+2)][nseg][NB]
    float *red = partial + (size_t)(geo.maxTileRows + 2) * nseg * NB;        // [32]: 16 reduction slots + 16 arg-max indices
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(red + 32);             // [nStages]
    uint64_t *emptyBar = fullBar + kMaxStages;                              // [nStages]

    traceStamp(a.trace, 0);
    pdlLaunchDependents();
    if (tid == 0) {
        for (uint32_t s = 0; s < geo.nStages; s++) {
            mbarInit(&fullBar[s], 1);
            mbarInit(&emptyBar[s], kConsumerWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // =============================== producer ===============================
        if (lane == 0) {
            const uint8_t *qsBase = reinterpret_cast<const uint8_t *>(a.qs);
            const uint8_t *scBase = reinterpret_cast<const uint8_t *>(a.scales);
            if (moe) {
                pdlWait();   // the expert choice is produced by the router kernel
                const uint32_t e = (uint32_t)a.expertIdx[slot] - a.moeFirstExpert;
                if (e >= a.moeNumLocal) return;   // expert lives on another rank (expert parallelism): nothing to stream
                qsBase += (uint64_t)e * a.expertQsStride * 4;
                scBase += (uint64_t)e * a.expertScaleStride * 2;
            }
            const uint64_t policy = policyEvictFirst();
            uint32_t st = 0, par = 0;
            bool wrapped = false;
            for (uint32_t f = 0; f < nFills; f++) {
                if (wrapped) mbarWait(&emptyBar[st], par ^ 1u);
                const uint32_t r0 = f * SR;
                const uint32_t rows = min(SR, tileRows - r0);
                const uint32_t bq = rows * rowQsBytes, bs = rows * rowScBytes;
                uint8_t *dst = ring + (size_t)st * geo.stageBytes;
                mbarExpectTx(&fullBar[st], bq + bs);
                tmaBulkLoad(dst, qsBase + (uint64_t)(rowBase + r0) * rowQsBytes, bq, &fullBar[st], policy);
                tmaBulkLoad(dst + (size_t)SR * rowQsBytes, scBase + (uint64_t)(rowBase + r0) * rowScBytes, bs, &fullBar[st], policy);
                if (++st == geo.nStages) { st = 0; par ^= 1u; wrapped = true; }
            }
        }
        return;
    }

    // =============================== consumers ===============================
    // norm weights are constants: pull them towards L2 while we wait for the predecessor
    if (PRO == PRO_RMSNORM_) {
        for (uint32_t i = tid * 32; i < a.n; i += kConsumerThreads * 32)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.normW + i));
    }
    pdlWait();
    traceStamp(a.trace, 1);
    const bool active = !moe || ((uint32_t)a.expertIdx[slot] - a.moeFirstExpert) < a.moeNumLocal;
    const float *inBase = a.in + (size_t)slot * a.inSlotStride;

    // ---- prologue: (rmsnorm) + q80 quantisation into the dp4a plane layout ----
    if (active) {
        const uint32_t nVec = a.n / 4;
#pragma unroll 1
        for (int t = 0; t < NB; t++) {
            const float4 *x4 = reinterpret_cast<const float4 *>(inBase + (size_t)t * a.inStride);
            float inv = 1.f;
            if (PRO == PRO_RMSNORM_) {
                float ss = 0.f;
                for (uint32_t i = tid; i < nVec; i += kConsumerThreads) {
                    const float4 v = x4[i];
                    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
                }
                ss = consumerSum(ss, red);
                inv = rsqrtf(ss / (float)a.n + a.eps);
            }
            uint8_t *pa = reinterpret_cast<uint8_t *>(planeA + (size_t)t * nblk);
            uint8_t *pb = reinterpret_cast<uint8_t *>(planeB + (size_t)t * nblk);
            for (uint32_t base = 0; base < nVec; base += kConsumerThreads) {
                const uint32_t i = base + tid;
                const bool act = i < nVec;
                float4 v = act ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                if (PRO == PRO_RMSNORM_ && act) v = rmsScale(v, reinterpret_cast<const float4 *>(a.normW)[i], inv);
                q80Pack(v, i, act, pa, pb, dxs + (size_t)t * nblk, dx8 + (size_t)t * nblk);
            }
        }
    }
    consumerBarrier();
    traceStamp(a.trace, 2);

    // ---- main loop over ring stages ----
    // stage index / parity / step rotation are carried incrementally: no integer division inside the fill loop
    const uint32_t stepsPerFullStage = (SR / kRowsPerStep) * nseg;
    const uint32_t rotInc = stepsPerFullStage % kConsumerWarps;
    const uint32_t gInc = kConsumerWarps / nseg, segInc = kConsumerWarps - gInc * nseg;
    const uint32_t recipNseg = 65536u / nseg + 1u;   // (s * recip) >> 16 == s / nseg for s < 16 while s * nseg < 2^16 (nseg < 4096)
    uint32_t st = 0, par = 0, rot = 0;
    for (uint32_t f = 0; active && f < nFills; f++) {
        const uint32_t r0 = f * SR;
        const uint32_t rows = min(SR, tileRows - r0);
        const uint32_t nGroups = (rows + kRowsPerStep - 1) / kRowsPerStep;
        const uint32_t nSteps = nGroups * nseg;
        const uint8_t *stage = ring + (size_t)st * geo.stageBytes;
        const uint4 *sq = reinterpret_cast<const uint4 *>(stage);
        const uint16_t *ss = reinterpret_cast<const uint16_t *>(stage + (size_t)SR * rowQsBytes);
        // steps are dealt round-robin over the 16 warps *across* fills (a stage may hold fewer than 16 steps)
        const uint32_t firstStep = ((uint32_t)warp - rot) & (kConsumerWarps - 1);
        rot = (rot + rotInc) & (kConsumerWarps - 1);
        // every warp waits (even one without steps in this fill): it keeps all warps within one ring revolution, so no
        // warp can arrive twice on the same empty-barrier phase
        mbarWait(&fullBar[st], par);
        uint32_t g = (firstStep * recipNseg) >> 16, seg = firstStep - g * nseg;
        for (uint32_t s = firstStep; s < nSteps; s += kConsumerWarps) {
            const uint32_t blk = seg * 32 + lane;
            const uint32_t rl = g * kRowsPerStep;                  // first row of the group inside the stage
            float acc[kRowsPerStep][NB];
            stageStepDot<NB>(sq, ss, rl, blk, nblk, planeA, planeB, dxs, dx8, acc);
#pragma unroll
            for (int t = 0; t < NB; t++) {
                const float v = reduce4(acc[0][t], acc[1][t], acc[2][t], acc[3][t], lane);
                if ((lane & 7) == 0) {
                    const uint32_t r = lane >> 3;
                    if (rl + r < rows) partial[((r0 + rl + r) * nseg + seg) * NB + t] = v;
                }
            }
            g += gInc;
            seg += segInc;
            if (seg >= nseg) { seg -= nseg; g++; }
        }
        __syncwarp();
        if (lane == 0) mbarArrive(&emptyBar[st]);
        if (++st == geo.nStages) { st = 0; par ^= 1u; }
    }
    consumerBarrier();

    // ---- epilogue ----
    auto rowSum = [&](uint32_t r, uint32_t t) { return segRowSum<NB>(partial, r, t, nseg); };
    if (EPI == EPI_SWIGLU_) {
        const uint32_t tilePairs = tileRows / 2;
        float *outBase = a.out + (size_t)slot * a.outSlotStride;
        for (uint32_t i = tid; i < tilePairs * NB; i += kConsumerThreads) {
            const uint32_t p = i / NB, t = i - p * NB;
            outBase[(size_t)t * a.outStride + pairBegin + p] = active ? gateAct(rowSum(2 * p, t), a.act) * rowSum(2 * p + 1, t) : 0.f;
        }
    } else if (EPI == EPI_RESIDUAL_ || EPI == EPI_MOE_DOWN_) {
        __shared__ bool sLastSlot;
        if (EPI == EPI_MOE_DOWN_) {
            // every routing slot leaves its weighted product in the scratch; the last slot CTA of a row tile sums the
            // slots in fixed order (deterministic) and carries on with the residual add / all-reduce
            const float wgt = active ? a.expertWeight[slot] : 0.f;
            for (uint32_t i = tid; i < tileRows; i += kConsumerThreads)
                a.moeScratch[(size_t)slot * a.d + rowBase + i] = active ? rowSum(i, 0) * wgt : 0.f;
            __threadfence();
            consumerBarrier();
            if (tid == 0) {
                const unsigned int prev = atomicAdd(&a.moeCounters[tileIdx], 1u);
                sLastSlot = prev == a.kActive - 1;
                if (sLastSlot) a.moeCounters[tileIdx] = 0;
            }
            consumerBarrier();
            if (!sLastSlot) { traceStamp(a.trace, 3); return; }
            __threadfence();
        }
        auto value = [&](uint32_t r, uint32_t t) {
            if (EPI == EPI_MOE_DOWN_) {
                float v = 0.f;
                for (uint32_t j = 0; j < a.kActive; j++) v += __ldcg(a.moeScratch + (size_t)j * a.d + rowBase + r);
                return v;
            }
            return rowSum(r, t);
        };
        if (a.ar.nRanks > 1) {
            // ---- fused one-shot all-reduce over NVLink peer memory + residual add -------------------------------
            // Every rank computed the partial product of the same row tile in the CTA with the same index. LL protocol:
            // every 8-byte word carries (partial value, valid flag); the partial rows are stored into slot[myRank] of
            // *every* rank, receivers poll the words of all sources, sum them in rank order (bit-identical result on
            // every rank) and clear them for the all-reduce after next (the slots are double buffered by parity).
            const ArArgs &ar = a.ar;
            const size_t slotBase = (size_t)(ar.parity * ar.nRanks + ar.rank) * ar.slotStride;
            for (uint32_t i = tid; i < tileRows * NB; i += kConsumerThreads) {
                const uint32_t r = i / NB, t = i - r * NB;
                const float v = value(r, t);
                const size_t off = slotBase + (size_t)t * ar.dim + rowBase + r;
#pragma unroll 1
                for (uint32_t p = 0; p < ar.nRanks; p++) stLL(ar.slots[(ar.rank + p) % ar.nRanks] + off, __float_as_uint(v), 1u);
            }
            uint64_t *mine = ar.slots[ar.rank];
            for (uint32_t i = tid; i < tileRows * NB; i += kConsumerThreads) {
                const uint32_t r = i / NB, t = i - r * NB;
                float sum = 0.f;
                for (uint32_t sr = 0; sr < ar.nRanks; sr++) {
                    uint64_t *w = mine + (size_t)(ar.parity * ar.nRanks + sr) * ar.slotStride + (size_t)t * ar.dim + rowBase + r;
                    uint2 v = ldLL(w);
                    while (v.y == 0u) v = ldLL(w);
                    sum += __uint_as_float(v.x);
                    stLL(w, 0u, 0u);
                }
                a.out[(size_t)t * a.outStride + rowBase + r] += sum;
            }
        } else {
            for (uint32_t i = tid; i < tileRows * NB; i += kConsumerThreads) {
                const uint32_t r = i / NB, t = i - r * NB;
                a.out[(size_t)t * a.outStride + rowBase + r] += value(r, t);
            }
        }
    } else {
        float best = -INFINITY;
        int bestIdx = 0x7fffffff;
        for (uint32_t i = tid; i < tileRows * NB; i += kConsumerThreads) {
            const uint32_t r = i / NB, t = i - r * NB;
            const float v = rowSum(r, t);
            a.out[(size_t)t * a.outStride + rowBase + r] = v;
            if ((EPI == EPI_ARGMAX_ || EPI == EPI_ARGMAX_ROWS_) && v > best && a.rowOffsetGlobal + rowBase + r < a.vocabLimit) { best = v; bestIdx = (int)(a.rowOffsetGlobal + rowBase + r); }   // rows ascend per thread
        }
        if (EPI == EPI_ARGMAX_) {
            // greedy sampling fused into the logits kernel: the next token and the position advance stay on the device
            const ArgMaxOut o{a.argVal, a.argIdx, a.argCounter, a.tokenOut, a.posInOut, a.history, a.historyCap};
            argMaxEpilogue(best, bestIdx, red, o, a.ar, tid, [] { return false; });
        }
        if constexpr (EPI == EPI_ARGMAX_ROWS_ && NB > 1) {
            // a thread's rows all belong to logits row tid % NB; the activation planes are no longer read
            const ArgMaxOut o{a.argVal, a.argIdx, a.argCounter, a.tokenOut, nullptr, nullptr, 0};
            argMaxRowsEpilogue<NB>(best, bestIdx, reinterpret_cast<float *>(planeA), o, tid);
        }
    }
    traceStamp(a.trace, 3);
}

// Whether gemvQ40TmaKernel (tma) or gemvQ40Kernel is compiled for (pro, epi, nb).
static bool instantiated(bool tma, int pro, int epi, int nb) {
#define DL_LISTED(P, E, N) \
    if (pro == P && epi == E && nb == N) return true;
    if (tma) {
        DL_GEMV_Q40_TMA_INSTANCES(DL_LISTED)
    } else {
        DL_GEMV_Q40_LDG_INSTANCES(DL_LISTED)
    }
#undef DL_LISTED
    return false;
}

// TMA-ring plan of one launch; rc 1 when the shape cannot use the TMA path.
static GemvQ40Plan planTma(int pro, int epi, int nb, uint32_t d, uint32_t n, int numSms, uint32_t moeCtasPerSlot, uint32_t kActive) {
    GemvQ40Plan p{};
    p.launches = 1;
    if (d % 2 || n % 128) { p.rc = 1; return p; }   // bulk copies need 16-byte aligned row starts for the fp16 scale rows
    const uint32_t nblk = n / 32, nseg = (nblk + 31) / 32;
    const uint32_t nPairs = d / 2;
    uint32_t grid = nPairs < (uint32_t)numSms ? nPairs : (uint32_t)numSms;
    uint32_t tilesPerMatrix = grid;
    if (moeCtasPerSlot) {
        if (nb != 1) { p.rc = -4; return p; }
        tilesPerMatrix = moeCtasPerSlot;
        grid = moeCtasPerSlot * kActive;
    }
    const uint32_t maxTileRows = 2 * ((nPairs + tilesPerMatrix - 1) / tilesPerMatrix);
    const uint32_t rowBytes = nblk * 18;
    // a stage should hold >= 16 steps (one per consumer warp) so the per-stage barrier traffic is amortised
    uint32_t sr = (64 + nseg - 1) / nseg;
    sr = (sr + 3) / 4 * 4;
    while (sr > 4 && sr * rowBytes > 36 * 1024) sr -= 4;
    if (sr * rowBytes > 48 * 1024) { p.rc = 1; return p; }   // rows too wide for a 4-row stage: per-thread-load kernel handles it
    if (sr > 64) sr = 64;
    const uint32_t stageBytes = (sr * rowBytes + 127) / 128 * 128;
    const size_t fixedBytes = (size_t)nb * nblk * (16 + 16 + 4 + 4) + (size_t)(maxTileRows + 2) * nseg * nb * 4 + 32 * 4 +
                              2 * kMaxStages * 8 + 256;
    const size_t budget = (nb == 1 ? 112 : 226) * 1024;   // nb == 1: leave room for the next kernel's CTA on the same SM
    if (fixedBytes + stageBytes > budget) { p.rc = 1; return p; }
    uint32_t stages = (uint32_t)((budget - fixedBytes) / stageBytes);
    const uint32_t need = (maxTileRows + sr - 1) / sr;
    if (stages > need) stages = need;
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 1) { p.rc = 1; return p; }
    if (!instantiated(true, pro, epi, nb)) { p.rc = -3; return p; }
    p.kernel = 2;
    p.grid = grid;
    p.maxTileRows = maxTileRows;
    p.stageRows = sr;
    p.nStages = stages;
    p.smemBytes = (uint32_t)(fixedBytes + (size_t)stages * stageBytes);
    return p;
}

GemvQ40Plan planGemvQ40(int pro, int epi, int nb, uint32_t d, uint32_t n, int numSms, int impl, bool split, uint32_t moeCtasPerSlot,
                        uint32_t kActive) {
    if (impl != 1) {
        const GemvQ40Plan t = planTma(pro, epi, nb, d, n, numSms, moeCtasPerSlot, kActive);
        if (t.rc != 1 || impl == 2) return t;
    }
    GemvQ40Plan p{};
    p.launches = 1;
    if (d % 2 || n % 32 || (n / 4) % 8) { p.rc = -1; return p; }
    const uint32_t nPairs = d / 2;
    p.grid = nPairs < (uint32_t)numSms ? nPairs : (uint32_t)numSms;
    p.maxTileRows = 2 * ((nPairs + p.grid - 1) / p.grid);
    const size_t smemBytes = gemvSmemBytes(n, p.maxTileRows, nb);
    if (smemBytes > 227 * 1024) {
        // no kernel holds nb tokens: the tokens of STORE / RESIDUAL / SWIGLU are independent, so two launches of nb / 2 are exact
        if (split && nb > 1 && moeCtasPerSlot == 0 && (epi == EPI_STORE_ || epi == EPI_RESIDUAL_ || epi == EPI_SWIGLU_)) {
            GemvQ40Plan h = planGemvQ40(pro, epi, nb / 2, d, n, numSms, impl, split);
            if (h.rc == 0) {
                h.launches *= 2;
                return h;
            }
        }
        p.rc = -2;
        return p;
    }
    if (!instantiated(false, pro, epi, nb)) { p.rc = -3; return p; }
    p.kernel = 1;
    p.smemBytes = (uint32_t)smemBytes;
    return p;
}

int launchGemvQ40Tma(int pro, int epi, int nb, GemvArgs a, const GemvQ40Plan &p, cudaStream_t stream, bool pdl) {
    a.act = gHiddenAct;
    if (a.vocabLimit == 0) a.vocabLimit = 0xffffffffu;
    TmaGemvGeom geo{};
    geo.maxTileRows = p.maxTileRows;
    geo.stageRows = p.stageRows;
    geo.nStages = p.nStages;
    geo.stageBytes = (p.stageRows * (a.n / 32) * 18 + 127) / 128 * 128;
#define DL_LAUNCH(P, E, N)                                                                                                        \
    if (pro == P && epi == E && nb == N) {                                                                                        \
        DL_CUDA_CHECK((raiseSmemLimit<gemvQ40TmaKernel<P, E, N>>(p.smemBytes)));                                                  \
        DL_CUDA_CHECK((launchPdl(gemvQ40TmaKernel<P, E, N>, dim3(p.grid), dim3(kTmaThreads), p.smemBytes, stream, pdl, a, geo))); \
        return 0;                                                                                                                 \
    }
    DL_GEMV_Q40_TMA_INSTANCES(DL_LAUNCH)
#undef DL_LAUNCH
    return -3;
}

int gemvQ40Run(int pro, int epi, int nb, const GemvArgs &a, int numSms, cudaStream_t stream, bool pdl, int impl) {
    const bool split = a.ar.nRanks <= 1 && a.expertIdx == nullptr;
    const GemvQ40Plan p = planGemvQ40(pro, epi, nb, a.d, a.n, numSms, impl, split, a.moeCtasPerSlot, a.kActive);
    if (p.rc != 0) return p.rc;
    const int sub = nb / (int)p.launches;
    for (uint32_t i = 0; i < p.launches; i++) {
        GemvArgs s = a;
        s.in = a.in + (size_t)i * sub * a.inStride;
        s.out = a.out + (size_t)i * sub * a.outStride;
        const int r = p.kernel == 2 ? launchGemvQ40Tma(pro, epi, sub, s, p, stream, pdl) : launchGemvQ40Ldg(pro, epi, sub, s, p, stream, pdl);
        if (r != 0) return r;
    }
    return 0;
}

}  // namespace dl
