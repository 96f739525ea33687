// Persistent single-token decode kernel: one launch per generated token for dense models (Llama / Qwen3).
//
// The multi-kernel decode path pays a grid-completion latency at each of its 161 kernel boundaries and restarts the
// weight stream at every launch. Here one CTA per SM stays resident for the whole token:
//   * warp 16 (producer) walks the list of all weight matrices of the token and streams this CTA's row tile of each one
//     through a single shared-memory ring with cp.async.bulk + mbarriers; between a layer's QKV and WO fills it streams the
//     cached K/V rows of this CTA's attention items the same way. It never synchronises with the phases — only ring space
//     limits it — so the HBM stream runs continuously across phase boundaries and layers.
//   * warps 0-15 (consumers) execute the phases embedding -> per layer [QKV GEMV, attention | WO GEMV + residual |
//     W1|W3 GEMV + SwiGLU | W2 GEMV + residual] -> logits GEMV + arg-max, separated by software grid barriers (none between
//     QKV and attention: attention polls the q|k|v words of its own heads).
//   * Every vector that crosses a phase boundary (x, q|k|v, z, h) travels as LL words: 8-byte {f32 payload, epoch} stores that
//     L2 delivers atomically. The barrier therefore needs NO memory fence (a relaxed arrive + relaxed poll): it only orders
//     control flow, and a consumer that finds a word with a stale epoch simply re-reads it. With the weight stream running a
//     fenced barrier costs more than a relaxed one (tools/microbench_barrier.py): MEMBAR.GPU queues behind the
//     bulk-copy reads each SM keeps in flight. LL words *instead of* barriers lose (every thread
//     polling during the arrival skew floods L2); here the poll starts only after the arrival counter
//     says the stores have been issued, so it almost always succeeds on the first read.
//   * tensor-parallel runs use the same LL-word protocol between GPUs in the WO / W2 epilogues (one multimem.st through the
//     NVSwitch multicast mapping reaches every rank; unicast peer stores when no multicast object exists) and the cross-rank
//     arg-max.
// The kernel takes over the roles of NnExecutor's step loop + barriers (reference src/nn/nn-executor.cpp:137-175) on the GPU.
#include <type_traits>

#include "gemv_common.cuh"

namespace dl {

enum { MP_QKV = 0, MP_WO = 1, MP_W13 = 2, MP_W2 = 3, MP_LOGITS = 4 };   // index into MegaArgs::ph

static uint32_t megaStageRows(uint32_t n, uint32_t stageBytes) {
    const uint32_t rowBytes = (n / 32) * 18;
    uint32_t sr = stageBytes / rowBytes;
    sr = sr / 4 * 4;
    return sr > 64 ? 64 : sr;
}

struct MegaSmem {
    uint8_t *ring;
    uint4 *planeA, *planeB;
    float *dxs, *dx8, *partial, *red, *rope, *qHand;
    uint64_t *fullBar, *emptyBar;
};

// Spin budget of every wait loop in this kernel: a peer rank that died or a CTA that never became resident must not wedge the GPU.
// After ~2^27 polls (seconds) the waiter raises the abort flag (host-visible); every loop also leaves as soon as the flag is up,
// so the kernel drains and the host reports the failure (reference: socket exceptions, src/nn/nn-network.cpp:84-123).
constexpr uint32_t kSpinCheck = 1u << 12;
constexpr uint32_t kSpinLimit = 1u << 27;

struct SpinGuard {
    volatile unsigned int *abortFlag;
    uint32_t n = 0;
    __device__ __forceinline__ explicit SpinGuard(unsigned int *f) : abortFlag(f) {}
    // returns true when the caller must stop waiting
    __device__ __forceinline__ bool tick() {
        if ((++n & (kSpinCheck - 1)) != 0) return false;
        if (abortFlag && *abortFlag) return true;
        if (n >= kSpinLimit) {
            if (abortFlag) *abortFlag = 1u;
            return true;
        }
        return false;
    }
};

// Control-only grid barrier: relaxed arrive, relaxed poll. Data crossing it is self-validating (LL words), see the file header.
__device__ __forceinline__ void gridBarrier(unsigned int *ctr, unsigned int &target, int tid, unsigned int *abortFlag) {
    consumerBarrier();   // every consumer thread has issued its stores of this phase
    if (tid == 0) {
        asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
        target += gridDim.x;
        unsigned int v;
        SpinGuard g(abortFlag);
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        } while (v < target && !g.tick());
    }
    consumerBarrier();
}

// Fenced variant for the one boundary whose payload is too large for LL words (the 14336-long SwiGLU vector: as 8-byte words it
// costs every CTA 114 KB of L2 reads per layer, more than the fence): release/acquire make the plain f32 stores visible.
__device__ __forceinline__ void gridBarrierFenced(unsigned int *ctr, unsigned int &target, int tid, unsigned int *abortFlag) {
    consumerBarrier();
    if (tid == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
        target += gridDim.x;
        unsigned int v;
        SpinGuard g(abortFlag);
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        } while (v < target && !g.tick());
    }
    consumerBarrier();
}

// ---- LL words inside one GPU: {f32 payload, epoch} in one 8-byte store; readers compare the epoch ----
__device__ __forceinline__ void stW(uint2 *p, float v, uint32_t epoch) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(epoch) : "memory");
}
__device__ __forceinline__ uint4 ldW2(const uint2 *p) {   // two consecutive words
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint2 ldW(const uint2 *p) {
    uint2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
// One value, polled until its epoch matches.
__device__ __forceinline__ float ldWwait(const uint2 *p, uint32_t epoch, unsigned int *abortFlag) {
    uint2 v = ldW(p);
    if (v.y != epoch) {
        SpinGuard g(abortFlag);
        do { __nanosleep(100); v = ldW(p); } while (v.y != epoch && !g.tick());
    }
    return __uint_as_float(v.x);
}
// Four consecutive values (index i4 * 4 ..), polled until all four epochs match.
__device__ __forceinline__ float4 ldW4wait(const uint2 *base, uint32_t i4, uint32_t epoch, unsigned int *abortFlag) {
    const uint2 *p = base + (size_t)i4 * 4;
    uint4 a = ldW2(p), b = ldW2(p + 2);
    if (a.y != epoch || a.w != epoch || b.y != epoch || b.w != epoch) {
        SpinGuard g(abortFlag);
        do { __nanosleep(100); a = ldW2(p); b = ldW2(p + 2); } while ((a.y != epoch || a.w != epoch || b.y != epoch || b.w != epoch) && !g.tick());
    }
    return make_float4(__uint_as_float(a.x), __uint_as_float(a.z), __uint_as_float(b.x), __uint_as_float(b.z));
}

// Ring position shared (by construction) by the producer and the consumers: stage index + mbarrier phase parity, advanced
// once per fill. Kept incrementally — the hot loop contains no integer division (every `%`/`/` by a runtime value costs a
// ~20-instruction I2F/MUFU.RCP/F2I sequence per warp per fill, which used to dominate the per-fill overhead).
struct RingPos {
    uint32_t st, par;
    __device__ __forceinline__ void advance(uint32_t nStages) {
        if (++st == nStages) { st = 0; par ^= 1u; }
    }
};

// This CTA's pair-aligned row tile of a phase: the first `pairsRem` CTAs own one pair more (host-computed quotient/remainder).
__device__ __forceinline__ void megaTile(const MegaPhase &P, uint32_t &pairBegin, uint32_t &tileRows) {
    const uint32_t b = blockIdx.x;
    pairBegin = b * P.pairsQ + min(b, P.pairsRem);
    tileRows = 2 * (P.pairsQ + (b < P.pairsRem ? 1u : 0u));
}

// The producer's position in the token's weight stream: weight phase k (4 * layer + {QKV, WO, W1|W3, W2}, 4 * nLayers = logits)
// and row offset r0 inside this CTA's tile of it. Phases in which this CTA owns no rows are skipped, exactly as the consumers'
// main loops run zero fills there. One step of the cursor = one ring fill.
struct FillCursor {
    uint32_t k, r0;
    uint32_t tileRows, rowBase, SR, rowQsBytes, rowScBytes;
    const uint8_t *qs, *sc;

    __device__ __forceinline__ bool valid(const MegaArgs &m) const { return k <= 4 * m.nLayers; }
    // settle on the first phase >= k in which this CTA owns rows (r0 = 0)
    __device__ __forceinline__ void enter(const MegaArgs &m) {
        for (r0 = 0; k <= 4 * m.nLayers; k++) {
            const uint32_t l = k >> 2, w = k & 3;
            const MegaPhase &P = m.ph[l == m.nLayers ? (uint32_t)MP_LOGITS : w];
            uint32_t pairBegin;
            megaTile(P, pairBegin, tileRows);
            if (tileRows == 0) continue;
            rowBase = pairBegin * 2; SR = P.stageRows;
            rowQsBytes = P.nblk * 16; rowScBytes = P.nblk * 2;
            if (l == m.nLayers) { qs = m.wclsQs; sc = m.wclsSc; }
            else {
                const MegaLayer &L = m.layers[l];
                qs = w == MP_QKV ? L.qkvQs : w == MP_WO ? L.woQs : w == MP_W13 ? L.w13Qs : L.w2Qs;
                sc = w == MP_QKV ? L.qkvSc : w == MP_WO ? L.woSc : w == MP_W13 ? L.w13Sc : L.w2Sc;
            }
            return;
        }
    }
    __device__ __forceinline__ void next(const MegaArgs &m) {
        r0 += SR;
        if (r0 >= tileRows) { k++; enter(m); }
    }
    // source ranges of the current fill
    __device__ __forceinline__ uint32_t rows() const { return min(SR, tileRows - r0); }
    __device__ __forceinline__ const uint8_t *qsSrc() const { return qs + (uint64_t)(rowBase + r0) * rowQsBytes; }
    __device__ __forceinline__ const uint8_t *scSrc() const { return sc + (uint64_t)(rowBase + r0) * rowScBytes; }
};

// Attention work items: (head, split) pairs dealt round-robin to the CTAs (item blockIdx.x, + gridDim.x, ...). The producer derives
// the K/V fills of this CTA from the same rule as the consumers, so both must come from here.
constexpr uint32_t kKvChunk = kConsumerWarps * 4;   // cached K/V rows per ring fill: warp w takes rows 4w..4w+3
constexpr uint32_t kKvInflight = 2;                  // producer pacing of the K/V fills (the weight fills: MegaArgs::maxInflight)

// A q80 K/V fill (MegaArgs::kvScales set): the int8 K rows at stage offset 0, the V rows kKvChunk * HD bytes further, then the K and the V scale rows
// (HD / 16 bytes a row) in two regions of kvScRegion(HD) bytes. A bulk copy moves multiples of 16 bytes from 16-byte aligned
// addresses, so a fill copies the aligned span around its scale rows (the cache's scale planes carry 16 bytes of tail padding) and
// the consumers skip the leading kvScSkip bytes.
__host__ __device__ constexpr uint32_t kvScRegion(uint32_t hd) { return kKvChunk * hd / 16 + 16; }
__device__ __forceinline__ uint32_t kvScSkip(const void *firstRow) { return (uint32_t)(reinterpret_cast<uintptr_t>(firstRow) & 15u); }

// Effective split count: grows with the position (read on the device, so a replayed graph follows it), capped at nSplits.
__device__ __forceinline__ uint32_t attnSplits(const MegaArgs &m, uint32_t nPos) {
    uint32_t eff = (nPos + 255) / 256;
    if (eff > m.nSplits) eff = m.nSplits;
    if (eff < 1) eff = 1;
    return eff;
}
struct AttnItem {
    uint32_t h, split, kvh, begin, end, cachedEnd;   // cached rows [begin, cachedEnd) come through the ring
    bool ownsNew;                                     // the split that ends at the new position also takes this token's k/v
    __device__ __forceinline__ AttnItem(const MegaArgs &m, uint32_t item, uint32_t nPos, uint32_t eff) {
        h = item / eff; split = item - h * eff;
        kvh = h / (m.nHeads / m.nKvHeads);
        const uint32_t chunk = (nPos + eff - 1) / eff;
        begin = split * chunk;
        end = min(begin + chunk, nPos);
        ownsNew = end == nPos;
        cachedEnd = ownsNew ? end - 1 : end;
    }
};

// One GEMV phase on the consumer warps.
// `in` / inEpoch: LL vector consumed by the prologue; `outW` / outEpoch: LL vector produced by the epilogue (EPI_RESIDUAL: the
// residual stream itself, read-modify-written on the rows this CTA owns); `outF`: plain f32 output of the logits phase.
// IN_PLAIN: the input vector is plain f32 at `inF` (made visible by a fenced barrier) instead of LL words at `in`.
template <int PRO, int EPI, bool IN_PLAIN = false>
__device__ void megaGemv(const MegaArgs &m, const MegaSmem &sm, const MegaPhase &P, const uint2 *in, uint32_t inEpoch, const float *normW,
                         uint2 *outW, uint32_t outEpoch, float *outF, uint32_t arParity, RingPos &ring, int tid, uint32_t &slot,
                         const float *inF = nullptr, const uint2 *resW = nullptr) {
    auto stamp = [&]() { if (m.trace && tid == 0 && blockIdx.x < m.traceCtas) m.trace[(size_t)blockIdx.x * m.traceStride + slot] = globalTimerNs(); slot++; };
    const int lane = tid & 31, warp = tid >> 5;
    const uint32_t n = P.n;
    const uint32_t nblk = P.nblk, nseg = P.nseg;
    const uint32_t rowQsBytes = nblk * 16;
    uint32_t pairBegin, tileRows;
    megaTile(P, pairBegin, tileRows);
    const uint32_t rowBase = pairBegin * 2;
    const uint32_t SR = P.stageRows;
    uint4 *planeA = sm.planeA, *planeB = sm.planeB;
    float *dxs = sm.dxs, *dx8 = sm.dx8, *partial = sm.partial, *red = sm.red;

    // The residual of the rows this CTA owns is fetched now, so that its L2 round trip overlaps the prologue and the main loop
    // (own rows were written by this very thread in the previous residual phase / the embedding phase: no epoch check needed).
    float resid = 0.f;
    if (EPI == EPI_RESIDUAL_ && (uint32_t)tid < tileRows) resid = __uint_as_float(ldW((resW ? resW : outW) + rowBase + tid).x);

    // ---- prologue: (rmsnorm) + q80 quantisation of the activation vector. RMS-norm phases (n = dim <= 8192) keep the whole
    // vector in registers for the reduction; plain phases stream it in chunks of 16384 elements (any n) ----
    {
        const uint32_t nVec = n / 4;
        constexpr int kMaxVec = PRO == PRO_RMSNORM_ ? 4 : 8;
        constexpr uint32_t kChunkVec = kMaxVec * kConsumerThreads;
        uint8_t *pa = reinterpret_cast<uint8_t *>(planeA);
        uint8_t *pb = reinterpret_cast<uint8_t *>(planeB);
        for (uint32_t vecBase = 0; vecBase < nVec; vecBase += kChunkVec) {
            float4 xv[kMaxVec];
            float4 wv[PRO == PRO_RMSNORM_ ? kMaxVec : 1];
            if (PRO == PRO_RMSNORM_) {
#pragma unroll
                for (int k = 0; k < kMaxVec; k++) {
                    const uint32_t i = vecBase + k * kConsumerThreads + tid;
                    wv[k] = i < nVec ? __ldg(reinterpret_cast<const float4 *>(normW) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            float ss = 0.f;
            // NB: issuing the LL loads of several float4 before checking any epoch (one L2 round trip instead of one per value) was
            // rejected: the extra live registers push the 96-register kernel (17 warps are allocated as 20) into spilling
            // inside the dp4a main loop.
#pragma unroll
            for (int k = 0; k < kMaxVec; k++) {
                const uint32_t i = vecBase + k * kConsumerThreads + tid;
                if (IN_PLAIN) xv[k] = i < nVec ? __ldcg(reinterpret_cast<const float4 *>(inF) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                else xv[k] = i < nVec ? ldW4wait(in, i, inEpoch, m.abortFlag) : make_float4(0.f, 0.f, 0.f, 0.f);
                ss += xv[k].x * xv[k].x + xv[k].y * xv[k].y + xv[k].z * xv[k].z + xv[k].w * xv[k].w;
            }
            float inv = 1.f;
            if (PRO == PRO_RMSNORM_) {
                ss = consumerSum(ss, red);
                inv = rsqrtf(ss / (float)n + m.eps);
            }
#pragma unroll
            for (int k = 0; k < kMaxVec; k++) {
                const uint32_t i = vecBase + k * kConsumerThreads + tid;
                if (vecBase + k * kConsumerThreads >= nVec) break;     // block-uniform
                const bool act = i < nVec;
                float4 v = xv[k];
                if (PRO == PRO_RMSNORM_ && act) v = rmsScale(v, wv[PRO == PRO_RMSNORM_ ? k : 0], inv);
                q80Pack(v, i, act, pa, pb, dxs, dx8);
            }
        }
    }
    consumerBarrier();
    stamp();   // prologue done

    // ---- main loop over this phase's fills ----
    const uint32_t gInc = P.gInc, segInc = P.segInc;
    uint32_t rot = 0;   // (fill index * steps per full stage) mod 16: rotates the step -> warp assignment from fill to fill
    for (uint32_t r0 = 0; r0 < tileRows; r0 += SR) {
        const uint32_t st = ring.st;
        const uint32_t rows = min(SR, tileRows - r0);
        const uint32_t nSteps = ((rows + kRowsPerStep - 1) / kRowsPerStep) * nseg;
        const uint8_t *stage = sm.ring + st * m.stageBytes;
        const uint4 *sq = reinterpret_cast<const uint4 *>(stage);
        const uint16_t *ss = reinterpret_cast<const uint16_t *>(stage + SR * rowQsBytes);
        const uint32_t firstStep = ((uint32_t)warp - rot) & (kConsumerWarps - 1);
        rot = (rot + P.rotInc) & (kConsumerWarps - 1);
        uint32_t g = (firstStep * P.recipNseg) >> 16, seg = firstStep - g * nseg;   // firstStep / nseg, firstStep % nseg
        mbarWait(&sm.fullBar[st], ring.par);
        // two steps are processed together (independent dependency chains -> the LDS/IDP/SHFL latencies overlap)
        auto stepDot = [&](uint32_t g_, uint32_t seg_, float (&acc)[kRowsPerStep][1]) {
            stageStepDot<1>(sq, ss, g_ * kRowsPerStep, seg_ * 32 + lane, nblk, planeA, planeB, dxs, dx8, acc);
        };
        auto stepStore = [&](uint32_t g_, uint32_t seg_, float v) {
            const uint32_t rl = g_ * kRowsPerStep;
            if ((lane & 7) == 0) {
                const uint32_t r = lane >> 3;
                if (rl + r < rows) partial[(r0 + rl + r) * nseg + seg_] = v;
            }
        };
        auto advance = [&](uint32_t &g_, uint32_t &seg_) {
            g_ += gInc;
            seg_ += segInc;
            if (seg_ >= nseg) { seg_ -= nseg; g_++; }
        };
        uint32_t s = firstStep;
        for (; s + kConsumerWarps < nSteps; s += 2 * kConsumerWarps) {
            uint32_t g2 = g, seg2 = seg;
            advance(g2, seg2);
            float a0[kRowsPerStep][1], a1[kRowsPerStep][1];
            stepDot(g, seg, a0);
            stepDot(g2, seg2, a1);
            const float v0 = reduce4(a0[0][0], a0[1][0], a0[2][0], a0[3][0], lane);
            const float v1 = reduce4(a1[0][0], a1[1][0], a1[2][0], a1[3][0], lane);
            stepStore(g, seg, v0);
            stepStore(g2, seg2, v1);
            g = g2; seg = seg2;
            advance(g, seg);
        }
        if (s < nSteps) {
            float a0[kRowsPerStep][1];
            stepDot(g, seg, a0);
            stepStore(g, seg, reduce4(a0[0][0], a0[1][0], a0[2][0], a0[3][0], lane));
        }
        __syncwarp();
        if (lane == 0) mbarArrive(&sm.emptyBar[st]);
        ring.advance(m.nStages);
    }
    consumerBarrier();
    stamp();   // main loop done

    // ---- epilogue ----
    auto rowSum = [&](uint32_t r) { return segRowSum<1>(partial, r, 0, nseg); };
    if (EPI == EPI_SWIGLU_) {
        for (uint32_t p = tid; p < tileRows / 2; p += kConsumerThreads) outF[pairBegin + p] = gateAct(rowSum(2 * p), m.act) * rowSum(2 * p + 1);
    } else if (EPI == EPI_STORE_) {
        for (uint32_t r = tid; r < tileRows; r += kConsumerThreads) stW(outW + rowBase + r, rowSum(r), outEpoch);
    } else if (EPI == EPI_RESIDUAL_) {
        // tileRows <= kConsumerThreads (checked on the host): thread r owns row r of the tile
        if (m.ar.nRanks > 1) {
            const ArArgs &ar = m.ar;
            const size_t slotBase = (size_t)(arParity * ar.nRanks + ar.rank) * ar.slotStride;
            if ((uint32_t)tid < tileRows) {
                const uint32_t r = tid;
                const float v = rowSum(r);
                if (ar.slotsMc) {
                    // one store, replicated by the NVSwitch into slot[myRank] of every rank (this one included)
                    const uint64_t word = (uint64_t)__float_as_uint(v) | (1ull << 32);
                    asm volatile("multimem.st.relaxed.sys.global.b64 [%0], %1;" ::"l"(ar.slotsMc + slotBase + rowBase + r), "l"(word) : "memory");
                } else {
#pragma unroll 1
                    for (uint32_t p = 0; p < ar.nRanks; p++) stLL(ar.slots[(ar.rank + p) % ar.nRanks] + slotBase + rowBase + r, __float_as_uint(v), 1u);
                }
                uint64_t *mine = ar.slots[ar.rank];
                float sum = 0.f;
                SpinGuard g(m.abortFlag);
                const bool timeIt = m.syncNs && blockIdx.x == 0 && tid == 0;     // "Sync" time of the CLI lines: wait for the peers' partial sums
                const uint64_t tSync0 = timeIt ? globalTimerNs() : 0;
                // (requesting the N words in batches of 4 before examining them was slower at N = 8: kept sequential)
                for (uint32_t sr = 0; sr < ar.nRanks; sr++) {
                    uint64_t *w = mine + (size_t)(arParity * ar.nRanks + sr) * ar.slotStride + rowBase + r;
                    uint2 v2 = ldLL(w);
                    while (v2.y == 0u && !g.tick()) v2 = ldLL(w);
                    sum += __uint_as_float(v2.x);          // rank order: every rank computes the same sum
                    stLL(w, 0u, 0u);
                }
                if (timeIt) *m.syncNs += globalTimerNs() - tSync0;   // device-memory accumulator, touched by this one thread only
                stW(outW + rowBase + r, resid + sum, outEpoch);
            }
        } else if ((uint32_t)tid < tileRows) {
            stW(outW + rowBase + tid, resid + rowSum(tid), outEpoch);
        }
    } else {
        float best = -INFINITY;
        int bestIdx = 0x7fffffff;
        for (uint32_t r = tid; r < tileRows; r += kConsumerThreads) {
            const float v = rowSum(r);
            outF[rowBase + r] = v;
            if (EPI == EPI_ARGMAX_ && v > best && m.rowOffsetGlobal + rowBase + r < m.vocabLimit) { best = v; bestIdx = (int)(m.rowOffsetGlobal + rowBase + r); }
        }
        if (EPI == EPI_ARGMAX_) {
            const ArgMaxOut o{m.argVal, m.argIdx, m.argCounter, m.greedyAdvance ? m.tokens : nullptr, m.pos, m.history, m.seqLen};
            SpinGuard g(m.abortFlag);
            argMaxEpilogue(best, bestIdx, red, o, m.ar, tid, [&g] { return g.tick(); });
        }
    }
}

// Attention phase: work items (head, split) are dealt round-robin to the CTAs (AttnItem); the 16 consumer warps of a CTA share
// the positions of one item. Same math as attnFusedKernel (attn_decode.cu). The cached K/V rows of an item arrive through the ring,
// kKvChunk rows per fill (the producer issues them between this layer's QKV and WO fills), warp w takes rows 4w..4w+3 of each.
// The q|k|v words are polled by warp 0 alone, and q is handed to the other warps through shared memory: this phase follows the
// QKV epilogue without a grid barrier, so the poll covers the other CTAs' arrival skew.
template <int HD, bool Q8>
__device__ void megaAttention(const MegaArgs &m, const MegaSmem &sm, const MegaLayer &L, int p, int tid, uint32_t inEpoch, uint32_t outEpoch,
                             RingPos &ring) {
    constexpr int DPL = HD / 32;
    const int lane = tid & 31, warp = tid >> 5;
    const uint32_t nPos = (uint32_t)p + 1;
    const uint32_t eff = attnSplits(m, nPos);
    const uint32_t kvMul = m.nHeads / m.nKvHeads;
    const uint32_t qDim = m.nHeads * HD, kvDim = m.nKvHeads * HD;
    float *sAcc = sm.partial;                 // [16][HD]
    float *sM = sm.partial + 16 * HD;         // [16]
    float *sL = sM + 16;                      // [16]
    __shared__ bool sLast;
    // rotary table row of this token's position: staged in shared memory once per launch (it is the same for all layers)
    const float2 *ropeRow = reinterpret_cast<const float2 *>(sm.rope) + lane * (DPL / 2);
    auto normRope = [&](float *v, const float *nw) {
        if (nw) {
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) ss += v[i] * v[i];
            ss = warpSum(ss);
            const float inv = rsqrtf(ss / (float)HD + m.eps);
#pragma unroll
            for (int i = 0; i < DPL; i++) v[i] = nw[lane * DPL + i] * (v[i] * inv);
        }
#pragma unroll
        for (int k = 0; k < DPL / 2; k++) {
            const float2 cs = ropeRow[k];
            const float x0 = v[2 * k] * cs.x - v[2 * k + 1] * cs.y;
            const float x1 = v[2 * k] * cs.y + v[2 * k + 1] * cs.x;
            v[2 * k] = x0; v[2 * k + 1] = x1;
        }
    };
    for (uint32_t item = blockIdx.x; item < m.nHeads * eff; item += gridDim.x) {
        const AttnItem it(m, item, nPos, eff);
        const uint32_t h = it.h, split = it.split, kvh = it.kvh, cachedEnd = it.cachedEnd;
        const bool ownsNew = it.ownsNew;
        // (the bf16 path keeps its own pointer arithmetic: same code as before the q80 variant)
        using KvT = typename std::conditional<Q8, int8_t, __nv_bfloat16>::type;
        KvT *kHead = reinterpret_cast<KvT *>(L.kCache) + (size_t)kvh * m.seqLen * HD;
        KvT *vHead = reinterpret_cast<KvT *>(L.vCache) + (size_t)kvh * m.seqLen * HD;
        const MegaKvScales *lsc = Q8 ? m.kvScales + (&L - m.layers) : nullptr;
        __half *kSc = Q8 ? lsc->k + (size_t)kvh * m.seqLen * (HD / 32) : nullptr;
        __half *vSc = Q8 ? lsc->v + (size_t)kvh * m.seqLen * (HD / 32) : nullptr;
        constexpr int UN = 4;
        static_assert(kConsumerWarps * UN == kKvChunk, "one ring fill of K/V rows = one batch of the 16 warps");
        using RawT = typename std::conditional<DPL == 4, uint2, uint32_t>::type;   // DPL bf16 values of one cache row
        auto unpack = [&](const RawT &r, float (&o)[DPL]) {
            if constexpr (DPL == 4) {
                const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.x));
                const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.y));
                o[0] = a0.x; o[1] = a0.y; o[2] = a1.x; o[3] = a1.y;
            } else {
                const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r));
                o[0] = a0.x; o[1] = a0.y;
            }
        };
        // On the item that owns the new position, warp 0 requests the raw k/v words before it polls q: one L2 round trip, not two.
        const bool newRow = ownsNew && warp == 0;
        const uint2 *ksrc = m.qkvW + qDim + (size_t)kvh * HD + lane * DPL;
        const uint2 *vsrc = m.qkvW + qDim + kvDim + (size_t)kvh * HD + lane * DPL;
        float q[DPL], kn[DPL], vn[DPL];
        if (warp == 0) {
            const uint2 *src = m.qkvW + (size_t)h * HD + lane * DPL;
            if constexpr (DPL == 4) {
                uint4 ka0, ka1, va0, va1;
                if (newRow) { ka0 = ldW2(ksrc); ka1 = ldW2(ksrc + 2); va0 = ldW2(vsrc); va1 = ldW2(vsrc + 2); }
                const float4 v = ldW4wait(src, 0, inEpoch, m.abortFlag);
                q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
                if (newRow) {
                    if (ka0.y != inEpoch || ka0.w != inEpoch || ka1.y != inEpoch || ka1.w != inEpoch || va0.y != inEpoch || va0.w != inEpoch ||
                        va1.y != inEpoch || va1.w != inEpoch) {
                        const float4 a = ldW4wait(ksrc, 0, inEpoch, m.abortFlag), bq = ldW4wait(vsrc, 0, inEpoch, m.abortFlag);
                        kn[0] = a.x; kn[1] = a.y; kn[2] = a.z; kn[3] = a.w;
                        vn[0] = bq.x; vn[1] = bq.y; vn[2] = bq.z; vn[3] = bq.w;
                    } else {
                        kn[0] = __uint_as_float(ka0.x); kn[1] = __uint_as_float(ka0.z); kn[2] = __uint_as_float(ka1.x); kn[3] = __uint_as_float(ka1.z);
                        vn[0] = __uint_as_float(va0.x); vn[1] = __uint_as_float(va0.z); vn[2] = __uint_as_float(va1.x); vn[3] = __uint_as_float(va1.z);
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < DPL; i++) q[i] = ldWwait(src + i, inEpoch, m.abortFlag);
                if (newRow) {
#pragma unroll
                    for (int i = 0; i < DPL; i++) { kn[i] = ldWwait(ksrc + i, inEpoch, m.abortFlag); vn[i] = ldWwait(vsrc + i, inEpoch, m.abortFlag); }
                }
            }
#pragma unroll
            for (int i = 0; i < DPL; i++) sm.qHand[lane * DPL + i] = q[i];
        }
        consumerBarrier();   // (the other warps read the previous item's q before that item's merge barriers)
        if (warp != 0) {
#pragma unroll
            for (int i = 0; i < DPL; i++) q[i] = sm.qHand[lane * DPL + i];
        }
        normRope(q, L.qNorm);
        const float scale = rsqrtf((float)HD);
#pragma unroll
        for (int i = 0; i < DPL; i++) q[i] *= scale;
        float mx = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
        for (int i = 0; i < DPL; i++) acc[i] = 0.f;
        if (newRow) {
            normRope(kn, L.kNorm);
            if constexpr (Q8) {
                const size_t e = (size_t)p * HD + lane * DPL;
                roundStoreKv<DPL, true>(kn, kHead, kSc, e, h % kvMul == 0);
                roundStoreKv<DPL, true>(vn, vHead, vSc, e, h % kvMul == 0);
            } else {
                __nv_bfloat162 kb[DPL / 2], vb[DPL / 2];
#pragma unroll
                for (int k = 0; k < DPL / 2; k++) {
                    kb[k] = __floats2bfloat162_rn(kn[2 * k], kn[2 * k + 1]);
                    vb[k] = __floats2bfloat162_rn(vn[2 * k], vn[2 * k + 1]);
                    const float2 kf = __bfloat1622float2(kb[k]), vf = __bfloat1622float2(vb[k]);
                    kn[2 * k] = kf.x; kn[2 * k + 1] = kf.y;
                    vn[2 * k] = vf.x; vn[2 * k + 1] = vf.y;
                }
                if (h % kvMul == 0) {
                    __nv_bfloat162 *kd = reinterpret_cast<__nv_bfloat162 *>(kHead + (size_t)p * HD + lane * DPL);
                    __nv_bfloat162 *vd = reinterpret_cast<__nv_bfloat162 *>(vHead + (size_t)p * HD + lane * DPL);
#pragma unroll
                    for (int k = 0; k < DPL / 2; k++) { kd[k] = kb[k]; vd[k] = vb[k]; }
                }
            }
            float dsum = 0.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) dsum += q[i] * kn[i];
            dsum = warpSum(dsum);
            mx = dsum; l = 1.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) acc[i] = vn[i];
        }
        // one ring fill per kKvChunk cached rows: K rows at the start of the stage, V rows kKvChunk rows further
        for (uint32_t c0 = it.begin; c0 < cachedEnd; c0 += kKvChunk) {
            const uint32_t st = ring.st;
            const uint8_t *stage = sm.ring + st * m.stageBytes;
            const __nv_bfloat16 *sK = reinterpret_cast<const __nv_bfloat16 *>(stage) + warp * UN * HD + lane * DPL;
            const __nv_bfloat16 *sV = sK + kKvChunk * HD;
            const uint32_t cur = c0 + warp * UN;
            mbarWait(&sm.fullBar[st], ring.par);
            float kf[UN][DPL], vf[UN][DPL];
            if constexpr (Q8) {
                // the rows and their scales as the producer placed them (see kvScRegion)
                const int8_t *sK8 = reinterpret_cast<const int8_t *>(stage);
                const __half *sKs = reinterpret_cast<const __half *>(stage + 2 * kKvChunk * HD + kvScSkip(kSc + (size_t)c0 * (HD / 32)));
                const __half *sVs = reinterpret_cast<const __half *>(stage + 2 * kKvChunk * HD + kvScRegion(HD) + kvScSkip(vSc + (size_t)c0 * (HD / 32)));
                const size_t e0 = (size_t)warp * UN * HD + lane * DPL;
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (cur + u < cachedEnd) {
                        loadKv<DPL, true>(sK8, sKs, e0 + u * HD, kf[u]);
                        loadKv<DPL, true>(sK8 + kKvChunk * HD, sVs, e0 + u * HD, vf[u]);
                    } else {
#pragma unroll
                        for (int i = 0; i < DPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
                    }
                }
            } else {
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (cur + u < cachedEnd) {
                        unpack(*reinterpret_cast<const RawT *>(sK + u * HD), kf[u]);
                        unpack(*reinterpret_cast<const RawT *>(sV + u * HD), vf[u]);
                    } else {
#pragma unroll
                        for (int i = 0; i < DPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbarArrive(&sm.emptyBar[st]);   // the rows are in registers: release the stage before the math
            ring.advance(m.nStages);
            float sc[UN];
#pragma unroll
            for (int u = 0; u < UN; u++) {
                float dsum = 0.f;
#pragma unroll
                for (int i = 0; i < DPL; i++) dsum += q[i] * kf[u][i];
                sc[u] = warpSum(dsum);
            }
#pragma unroll
            for (int u = 0; u < UN; u++) {
                if (cur + u < cachedEnd) {
                    const float mNew = fmaxf(mx, sc[u]);
                    const float corr = __expf(mx - mNew);
                    const float pr = __expf(sc[u] - mNew);
                    l = l * corr + pr;
#pragma unroll
                    for (int i = 0; i < DPL; i++) acc[i] = acc[i] * corr + pr * vf[u][i];
                    mx = mNew;
                }
            }
        }
        consumerBarrier();   // sAcc may still be read by the previous item
#pragma unroll
        for (int i = 0; i < DPL; i++) sAcc[warp * HD + lane * DPL + i] = acc[i];
        if (lane == 0) { sM[warp] = mx; sL[warp] = l; }
        consumerBarrier();
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < kConsumerWarps; w++) M = fmaxf(M, sM[w]);
        float num = 0.f, Lsum = 0.f;
        if (tid < HD) {
#pragma unroll
            for (int w = 0; w < kConsumerWarps; w++) {
                const float wgt = (sM[w] == -INFINITY) ? 0.f : __expf(sM[w] - M);
                num += sAcc[w * HD + tid] * wgt;
                Lsum += sL[w] * wgt;
            }
        }
        uint2 *outRow = m.zW + (size_t)h * HD;
        if (eff == 1) {
            if (tid < HD) stW(outRow + tid, num / Lsum, outEpoch);
            continue;
        }
        float *pOut = m.attnPartial + ((size_t)h * m.nSplits + split) * (HD + 2);
        if (tid < HD) pOut[tid] = num;
        if (tid == 0) { pOut[HD] = M; pOut[HD + 1] = Lsum; }
        __threadfence();
        consumerBarrier();
        if (tid == 0) {
            const unsigned int prev = atomicAdd(&m.attnCounters[h], 1u);
            sLast = (prev == eff - 1);
            if (sLast) m.attnCounters[h] = 0;
        }
        consumerBarrier();
        if (sLast) {
            __threadfence();
            const float *pIn = m.attnPartial + (size_t)h * m.nSplits * (HD + 2);
            float gM = -INFINITY;
            for (uint32_t s = 0; s < eff; s++) gM = fmaxf(gM, __ldcg(pIn + (size_t)s * (HD + 2) + HD));
            if (tid < HD) {
                float n2 = 0.f, den = 0.f;
                for (uint32_t s = 0; s < eff; s++) {
                    const float w = __expf(__ldcg(pIn + (size_t)s * (HD + 2) + HD) - gM);
                    n2 += w * __ldcg(pIn + (size_t)s * (HD + 2) + tid);
                    den += w * __ldcg(pIn + (size_t)s * (HD + 2) + HD + 1);
                }
                stW(outRow + tid, n2 / den, outEpoch);
            }
        }
    }
}

template <int HD, bool Q8>
__global__ void __launch_bounds__(kTmaThreads, 1) megaDecodeKernel(const __grid_constant__ MegaArgs m) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    MegaSmem sm;
    sm.ring = smem;
    sm.planeA = reinterpret_cast<uint4 *>(smem + (size_t)m.nStages * m.stageBytes);
    sm.planeB = sm.planeA + m.planeBlocks;
    sm.dxs = reinterpret_cast<float *>(sm.planeB + m.planeBlocks);
    sm.dx8 = sm.dxs + m.planeBlocks;
    sm.partial = sm.dx8 + m.planeBlocks;
    sm.red = sm.partial + m.partialFloats;
    sm.rope = sm.red + 32;                                              // [128] rotary (cos, sin) pairs of this token's position
    sm.qHand = sm.rope + 128;                                           // [128] attention: q of the item, polled by warp 0
    sm.fullBar = reinterpret_cast<uint64_t *>(sm.qHand + 128);
    sm.emptyBar = sm.fullBar + kMaxStages;

    if (tid == 0) {
        for (uint32_t s = 0; s < m.nStages; s++) {
            mbarInit(&sm.fullBar[s], 1);
            mbarInit(&sm.emptyBar[s], kConsumerWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // The position: read by every thread before the CTA's first barrier, since CTA 0 advances it at the end of the launch.
    int p = m.pos[0];
    if (p < 0) p = 0;
    if ((uint32_t)p >= m.seqLen) p = m.seqLen - 1;
    __syncthreads();

    if (warp == kConsumerWarps) {
        // =============================== producer: every weight matrix of the token, back to back ===============================
        if (lane == 0) {
            const uint64_t policy = policyEvictFirst();
            RingPos pr{0u, 0u};
            bool wrapped = false;   // every stage has been filled once: from now on wait for the consumers to free it
            // Pacing: at most `maxInflight` fills are outstanding at any time. The ring (capacity) still runs up to nStages
            // fills ahead of the consumers, but a freshly drained ring is refilled by a short pipeline of requests instead of
            // one ring-sized burst per SM: tens of MB of queued bulk reads chip-wide put microseconds of queueing delay in front
            // of every latency-critical load (barrier polls, activation vectors) at the L2 slices (tools/microbench_barrier.py).
            RingPos landed{0u, 0u};
            uint32_t nIssued = 0, nLanded = 0;
            const uint32_t maxInflight = m.maxInflight ? m.maxInflight : m.nStages;
            // K/V fills may have kKvInflight fills in flight (DESIGN.md §7): they are requested while the consumers still work on
            // QKV / W2, and their rows are cache reads of the kvMul q heads of a group rather than part of the weight stream.
            const uint32_t kvInflight = min(max(maxInflight, kKvInflight), m.nStages);
            auto waitLanded = [&](uint32_t cap) {
                while (nIssued - nLanded >= cap) {
                    mbarWait(&sm.fullBar[landed.st], landed.par);
                    landed.advance(m.nStages);
                    nLanded++;
                }
            };
            // All-CTA tracing: per weight phase, the ns spent waiting for a free stage (ring full) and on the in-flight cap, summed in
            // registers and stored once the fills move on to a later phase (phases without fills here store 0). The K/V fills of a
            // layer count towards its QKV phase.
            uint64_t *prodTrace = (m.trace && m.traceProdSlot && blockIdx.x < m.traceCtas)
                                      ? m.trace + (size_t)blockIdx.x * m.traceStride + m.traceProdSlot : nullptr;
            uint64_t fullNs = 0, capNs = 0;
            uint32_t traceK = 0;
            auto traceTo = [&](uint32_t k) {
                for (; traceK < k; traceK++) {
                    prodTrace[2 * traceK] = fullNs;
                    prodTrace[2 * traceK + 1] = capNs;
                    fullNs = capNs = 0;
                }
            };
            // one ring fill: wait for a free stage and for the in-flight count to drop under `cap`, then `copy(stage, full barrier)`
            auto fill = [&](uint32_t phaseK, uint32_t cap, uint32_t bytes, auto &&copy) {
                const uint32_t st = pr.st;
                if (prodTrace) {
                    traceTo(phaseK);
                    const uint64_t t0 = globalTimerNs();
                    if (wrapped) mbarWait(&sm.emptyBar[st], pr.par ^ 1u);
                    const uint64_t t1 = globalTimerNs();
                    waitLanded(cap);
                    const uint64_t t2 = globalTimerNs();
                    fullNs += t1 - t0;
                    capNs += t2 - t1;
                } else {
                    if (wrapped) mbarWait(&sm.emptyBar[st], pr.par ^ 1u);
                    waitLanded(cap);
                }
                nIssued++;
                mbarExpectTx(&sm.fullBar[st], bytes);
                copy(sm.ring + st * m.stageBytes, &sm.fullBar[st]);
                pr.advance(m.nStages);
                if (pr.st == 0) wrapped = true;
            };
            // K/V fills of layer l: this CTA's attention items (AttnItem, the consumers' rule), one fill per kKvChunk cached rows,
            // each fill = the K rows and the V rows (both contiguous in the head-major cache). Rows written by earlier launches only.
            const uint64_t kvPolicy = policyEvictNormal();   // a K/V row is read by the kvMul q heads of its group
            const uint32_t nPos = (uint32_t)p + 1, eff = attnSplits(m, nPos);
            auto kvFills = [&](uint32_t l) {
                const MegaLayer &L = m.layers[l];
                for (uint32_t item = blockIdx.x; item < m.nHeads * eff; item += gridDim.x) {
                    const AttnItem it(m, item, nPos, eff);
                    using KvT = typename std::conditional<Q8, int8_t, __nv_bfloat16>::type;
                    const KvT *kHead = reinterpret_cast<const KvT *>(L.kCache) + (size_t)it.kvh * m.seqLen * HD;
                    const KvT *vHead = reinterpret_cast<const KvT *>(L.vCache) + (size_t)it.kvh * m.seqLen * HD;
                    for (uint32_t c0 = it.begin; c0 < it.cachedEnd; c0 += kKvChunk) {
                        if constexpr (Q8) {
                            const uint32_t n = min(kKvChunk, it.cachedEnd - c0);
                            const size_t headOff = (size_t)it.kvh * m.seqLen * HD;
                            // int8 rows, then the 16-byte aligned span around their scale rows
                            const uint32_t bytes = n * HD;
                            const uint8_t *ks = reinterpret_cast<const uint8_t *>(m.kvScales[l].k + (headOff + (size_t)c0 * HD) / 32);
                            const uint8_t *vs = reinterpret_cast<const uint8_t *>(m.kvScales[l].v + (headOff + (size_t)c0 * HD) / 32);
                            const uint32_t kSkip = kvScSkip(ks), vSkip = kvScSkip(vs);
                            const uint32_t kSb = (kSkip + n * (HD / 16) + 15) & ~15u, vSb = (vSkip + n * (HD / 16) + 15) & ~15u;
                            fill(4 * l + MP_QKV, kvInflight, 2 * bytes + kSb + vSb, [&](uint8_t *dst, uint64_t *bar) {
                                tmaBulkLoad(dst, kHead + (size_t)c0 * HD, bytes, bar, kvPolicy);
                                tmaBulkLoad(dst + kKvChunk * HD, vHead + (size_t)c0 * HD, bytes, bar, kvPolicy);
                                tmaBulkLoad(dst + 2 * kKvChunk * HD, ks - kSkip, kSb, bar, kvPolicy);
                                tmaBulkLoad(dst + 2 * kKvChunk * HD + kvScRegion(HD), vs - vSkip, vSb, bar, kvPolicy);
                            });
                        } else {
                            const uint32_t bytes = min(kKvChunk, it.cachedEnd - c0) * HD * 2;
                            fill(4 * l + MP_QKV, kvInflight, 2 * bytes, [&](uint8_t *dst, uint64_t *bar) {
                                tmaBulkLoad(dst, kHead + (size_t)c0 * HD, bytes, bar, kvPolicy);
                                tmaBulkLoad(dst + kKvChunk * HD * 2, vHead + (size_t)c0 * HD, bytes, bar, kvPolicy);
                            });
                        }
                    }
                }
            };
            FillCursor cur;
            cur.k = 0;
            cur.enter(m);
            uint32_t kvLayer = 0;   // next layer whose K/V fills are due
            for (;;) {
                const bool more = cur.valid(m);
                // the consumers take a layer's K/V fills after its QKV fills and before any later phase's
                while (kvLayer < m.nLayers && (!more || cur.k > 4 * kvLayer)) kvFills(kvLayer++);
                if (!more) break;
                const uint32_t rows = cur.rows();
                const uint32_t bq = rows * cur.rowQsBytes, bs = rows * cur.rowScBytes;
                fill(cur.k, maxInflight, bq + bs, [&](uint8_t *dst, uint64_t *bar) {
                    tmaBulkLoad(dst, cur.qsSrc(), bq, bar, policy);
                    tmaBulkLoad(dst + cur.SR * cur.rowQsBytes, cur.scSrc(), bs, bar, policy);
                });
                cur.next(m);
            }
            if (prodTrace) traceTo(4 * m.nLayers + 1);
        }
        return;
    }

    // =============================== consumers ===============================
    unsigned int barTarget = 0;
    RingPos ring{0u, 0u};
    uint32_t slot = 0;
    auto stamp = [&]() { if (m.trace && tid == 0 && blockIdx.x < m.traceCtas) m.trace[(size_t)blockIdx.x * m.traceStride + slot] = globalTimerNs(); slot++; };
    stamp();
    // Epochs of the LL vectors: launch sequence number (device resident, bumped by CTA 0 at the end of every launch) x 1024 +
    // phase index. Phase indices: 0 = embedding; layer l: 1+5l QKV, 2+5l attention, 3+5l WO, 4+5l W1|W3, 5+5l W2.
    const uint32_t seqBase = __ldcg(m.launchSeq) << 10;
    if (tid < HD) sm.rope[tid] = m.rope[(size_t)p * HD + tid];
    // embedding: every CTA writes the rows of the residual stream it owns in the WO / W2 phases (same thread -> same rows, so
    // the residual read-modify-write never depends on another CTA's store)
    {
        int tok = m.tokens[0];
        if (tok < 0 || (uint32_t)tok >= m.vocabFull) tok = 0;
        uint32_t pairBegin, tileRows;
        megaTile(m.ph[MP_WO], pairBegin, tileRows);
        if ((uint32_t)tid < tileRows) stW(m.xW + pairBegin * 2 + tid, m.embedding.row((uint32_t)tok, m.dim)[pairBegin * 2 + tid], seqBase);
    }
    gridBarrier(m.gridCounter, barTarget, tid, m.abortFlag);
    // Experimental (MegaArgs::flags bit 0): no counter barrier where the consumer polls LL words anyway; the polls back off with
    // nanosleep. The residual stream alternates between two buffers so a fast CTA can never overwrite words a slow one still expects.
    const bool noBar = (m.flags & 1u) != 0;
    auto llBarrier = [&]() { if (!noBar) gridBarrier(m.gridCounter, barTarget, tid, m.abortFlag); };
    uint2 *xA = m.xW, *xB = noBar ? m.xW2 : m.xW;
    auto prefetchVec = [&](const float *p) {   // norm weights are constants: pull them towards L2 ahead of their phase
        for (uint32_t i = (blockIdx.x * kConsumerThreads + tid) * 32; i < m.dim; i += gridDim.x * kConsumerThreads * 32)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(p + i));
    };
    for (uint32_t l = 0; l < m.nLayers; l++) {
        const MegaLayer &L = m.layers[l];
        const uint32_t e0 = seqBase + 5 * l;     // epoch of x entering the layer (embedding or previous W2)
        prefetchVec(L.norm1);
        prefetchVec(l + 1 < m.nLayers ? m.layers[l + 1].norm0 : m.finalNorm);
        stamp();
        megaGemv<PRO_RMSNORM_, EPI_STORE_>(m, sm, m.ph[MP_QKV], xA, e0, L.norm0, m.qkvW, e0 + 1, nullptr, 0, ring, tid, slot);
        stamp();
        // no barrier: attention polls the q|k|v words it needs, CTAs without an attention item go on to the next barrier
        stamp();
        megaAttention<HD, Q8>(m, sm, L, p, tid, e0 + 1, e0 + 2, ring);
        stamp();
        llBarrier();
        stamp();
        megaGemv<PRO_PLAIN_, EPI_RESIDUAL_>(m, sm, m.ph[MP_WO], m.zW, e0 + 2, nullptr, xB, e0 + 3, nullptr, 0, ring, tid, slot, nullptr, xA);
        stamp();
        llBarrier();
        stamp();
        megaGemv<PRO_RMSNORM_, EPI_SWIGLU_>(m, sm, m.ph[MP_W13], xB, e0 + 3, L.norm1, nullptr, 0, m.hF, 0, ring, tid, slot);
        stamp();
        gridBarrierFenced(m.gridCounter, barTarget, tid, m.abortFlag);
        stamp();
        megaGemv<PRO_PLAIN_, EPI_RESIDUAL_, true>(m, sm, m.ph[MP_W2], nullptr, 0, nullptr, xA, e0 + 5, nullptr, 1, ring, tid, slot, m.hF, xB);
        stamp();
        llBarrier();
    }
    stamp();
    megaGemv<PRO_RMSNORM_, EPI_ARGMAX_>(m, sm, m.ph[MP_LOGITS], xA, seqBase + 5 * m.nLayers, m.finalNorm, nullptr, 0, m.logits, 0, ring, tid, slot);
    stamp();
    // every CTA has read launchSeq long ago (before its first barrier arrival): CTA 0 may advance it for the next launch
    if (blockIdx.x == 0 && tid == 0) *m.launchSeq = __ldcg(m.launchSeq) + 1u;
}

// Host: geometry + launch. Returns 1 if the model shape cannot use the persistent kernel.
int launchMegaDecode(MegaArgs m, int numSms, cudaStream_t stream) {
    if (m.headDim != 64 && m.headDim != 128) return 1;
    const uint32_t qDim = m.nHeads * m.headDim;
    const uint32_t ns[4] = {m.dim, qDim, m.ffDim, m.dim};
    uint32_t maxN = 0;
    for (uint32_t n : ns) {
        if (n % 128) return 1;
        if (n > maxN) maxN = n;
    }
    if (m.dim > 4 * kConsumerThreads * 4) return 1;   // RMS-norm phases keep the dim-long vector (+ norm weights) in registers
    if (5 * m.nLayers + 2 > 1023) return 1;           // phase index field of the LL epochs
    const uint32_t grid = (uint32_t)numSms;
    m.act = gHiddenAct;
    if (m.vocabLimit == 0) m.vocabLimit = 0xffffffffu;
    // partial buffer: rows of the largest tile x segments; also hosts the attention scratch (16 x HD + 32 floats)
    const uint32_t ds[5] = {qDim + 2 * m.nKvHeads * m.headDim, m.dim, 2 * m.ffDim, m.dim, m.vocab};
    const uint32_t dn[5] = {m.dim, qDim, m.dim, m.ffDim, m.dim};
    uint32_t partial = 16 * m.headDim + 64;
    for (int i = 0; i < 5; i++) {
        if (ds[i] % 2) return 1;
        const uint32_t tile = 2 * ((ds[i] / 2 + grid - 1) / grid) + 2;
        const uint32_t nseg = (dn[i] / 32 + 31) / 32;
        if (tile * nseg > partial) partial = tile * nseg;
    }
    m.partialFloats = (partial + 3) / 4 * 4;
    m.planeBlocks = maxN / 32;
    const size_t fixedBytes = (size_t)m.planeBlocks * (16 + 16 + 4 + 4) + (size_t)m.partialFloats * 4 + 32 * 4 + 2 * 128 * 4 + 2 * kMaxStages * 8 + 256;
    const size_t budget = 226 * 1024;
    // stage must hold >= 4 rows of the widest matrix
    const uint32_t maxRowBytes = (maxN / 32) * 18;
    uint32_t stageBytes = 36 * 1024;
    if (maxRowBytes * 4 > stageBytes) stageBytes = (maxRowBytes * 4 + 127) / 128 * 128;
    if (2 * kKvChunk * m.headDim * 2 > stageBytes) return 1;   // a K/V fill: kKvChunk bf16 rows of K and of V
    if (m.kvScales && 2 * kKvChunk * m.headDim + 2 * kvScRegion(m.headDim) > stageBytes) return 1;   // q80: int8 rows + scale spans
    if (fixedBytes + 2 * (size_t)stageBytes > budget) return 1;
    uint32_t stages = (uint32_t)((budget - fixedBytes) / stageBytes);
    if (stages > (uint32_t)kMaxStages) stages = kMaxStages;
    m.stageBytes = stageBytes;
    m.nStages = stages;
    // per-phase geometry, so the device code contains no integer division
    for (int i = 0; i < 5; i++) {
        MegaPhase &P = m.ph[i];
        P.d = ds[i]; P.n = dn[i];
        P.nblk = dn[i] / 32;
        P.nseg = (P.nblk + 31) / 32;
        P.stageRows = megaStageRows(dn[i], stageBytes);
        P.pairsQ = (ds[i] / 2) / grid;
        P.pairsRem = (ds[i] / 2) % grid;
        P.recipNseg = 65536u / P.nseg + 1u;                    // (s * recip) >> 16 == s / nseg for s < 16
        P.gInc = (uint32_t)kConsumerWarps / P.nseg;
        P.segInc = (uint32_t)kConsumerWarps - P.gInc * P.nseg;
        P.rotInc = ((P.stageRows / kRowsPerStep) * P.nseg) % (uint32_t)kConsumerWarps;
        for (uint32_t sft = 0; sft < (uint32_t)kConsumerWarps; sft++)
            if (((sft * P.recipNseg) >> 16) != sft / P.nseg) return 1;
    }
    // residual phases: thread r of a CTA owns row r of its tile
    if (2 * (m.ph[MP_WO].pairsQ + 1) > (uint32_t)kConsumerThreads) return 1;
    const size_t smemBytes = fixedBytes + (size_t)stages * stageBytes;
    // The kernel spins on grid barriers: every CTA must be resident at the same time. A cooperative launch makes the driver
    // verify that (and fail the launch instead of letting the barrier hang); the attribute cache is per device.
    const int v = (m.headDim == 128 ? 1 : 0) + (m.kvScales ? 2 : 0);
    int dev = 0;
    DL_CUDA_CHECK(cudaGetDevice(&dev));
    static size_t configured[16][4] = {};
    static int maxCoResident[16][4] = {};
    void (*const kernels[4])(MegaArgs) = {megaDecodeKernel<64, false>, megaDecodeKernel<128, false>, megaDecodeKernel<64, true>,
                                          megaDecodeKernel<128, true>};
    const void *fn = (const void *)kernels[v];
    const int d = dev & 15;
    if (smemBytes > configured[d][v]) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
        configured[d][v] = smemBytes;
        int perSm = 0, sms = 0;
        DL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, fn, kTmaThreads, smemBytes));
        DL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        maxCoResident[d][v] = perSm * sms;
    }
    if ((int)grid > maxCoResident[d][v]) return 1;   // would not be co-resident: the caller takes the multi-kernel path
    DL_CUDA_CHECK(cudaMemsetAsync(m.gridCounter, 0, sizeof(unsigned int), stream));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kTmaThreads);
    cfg.dynamicSmemBytes = smemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernels[v], m));
    return 0;
}

}  // namespace dl
