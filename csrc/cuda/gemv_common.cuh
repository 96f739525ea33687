// Device code shared by the decode GEMVs: the per-thread-load q40 kernel (gemv_q40.cu), the TMA-fed q40 kernel
// (gemv_q40_tma.cu), the persistent decode kernel's GEMV phases (mega_decode.cu) and the dense kernels (gemv_dense.cu).
// The q40 x q80 contract lives here once: the q80 rounding of the activation into the dp4a planes, the block dot product,
// the fixed-order row sums and the fused greedy arg-max.
#pragma once
#include "kernels.h"
#include "tma_common.cuh"

namespace dl {

// The compiled (PRO, EPI, NB) set of each q40 GEMV kernel: planGemvQ40 refuses (-3) what is not listed, and the launchers
// dispatch over the same list. X(PRO, EPI, NB) is expanded once per entry.
#define DL_GEMV_NB(X, P, E) X(P, E, 1) X(P, E, 2) X(P, E, 4) X(P, E, 8)
#define DL_GEMV_Q40_LDG_INSTANCES(X)                                                                                      \
    DL_GEMV_NB(X, PRO_RMSNORM_, EPI_STORE_) DL_GEMV_NB(X, PRO_PLAIN_, EPI_RESIDUAL_) DL_GEMV_NB(X, PRO_RMSNORM_, EPI_SWIGLU_) \
    DL_GEMV_NB(X, PRO_PLAIN_, EPI_STORE_) X(PRO_PLAIN_, EPI_SWIGLU_, 1)
#define DL_GEMV_Q40_TMA_INSTANCES(X) \
    DL_GEMV_Q40_LDG_INSTANCES(X) X(PRO_RMSNORM_, EPI_ARGMAX_, 1) X(PRO_PLAIN_, EPI_MOE_DOWN_, 1) \
    X(PRO_RMSNORM_, EPI_ARGMAX_ROWS_, 2) X(PRO_RMSNORM_, EPI_ARGMAX_ROWS_, 4) X(PRO_RMSNORM_, EPI_ARGMAX_ROWS_, 8)

// Sum over the 512 threads of a block; `red` holds 16 floats.
__device__ __forceinline__ float blockSum512(float v, float *red) {
    v = warpSum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < 16) ? red[lane] : 0.f;
    t = warpSum(t);
    __syncthreads();
    return t;
}

// RMS-norm scaling of four activations: w * (v * inv).
__device__ __forceinline__ float4 rmsScale(float4 v, float4 w, float inv) {
    return make_float4(w.x * (v.x * inv), w.y * (v.y * inv), w.z * (v.z * inv), w.w * (v.w * inv));
}

// Rounds v, elements 4i..4i+3 of an activation vector, to q80 (d = amax / 127 over the 32-element block, q = rint(x / d)) and
// stores it in the dp4a plane layout: quant block b = i / 8 takes 16 bytes of plane A, which pair with the low nibbles of
// the q40 words (common.cuh), and 16 bytes of plane B, which pair with the high nibbles. dxs[b] = f16(d), dx8[b] =
// 8 * f16(d) * sum(q) (the nibble bias). The 8 lanes of a block take part together (full-mask shuffles); lanes with
// act == false carry zeros and store nothing.
__device__ __forceinline__ void q80Pack(float4 v, uint32_t i, bool act, uint8_t *pa, uint8_t *pb, float *dxs, float *dx8) {
    float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
    const float d = amax / 127.f;
    const float id = d != 0.f ? 1.f / d : 0.f;
    const int q0 = __float2int_rn(v.x * id), q1 = __float2int_rn(v.y * id);
    const int q2 = __float2int_rn(v.z * id), q3 = __float2int_rn(v.w * id);
    int qsum = q0 + q1 + q2 + q3;
    qsum += __shfl_xor_sync(0xffffffffu, qsum, 1);
    qsum += __shfl_xor_sync(0xffffffffu, qsum, 2);
    qsum += __shfl_xor_sync(0xffffffffu, qsum, 4);
    if (act) {
        const uint32_t b = i >> 3, sub = i & 7, k = sub >> 1, odd = sub & 1;
        uint8_t *wa = pa + (size_t)b * 16 + k * 4 + odd;
        uint8_t *wb = pb + (size_t)b * 16 + k * 4 + odd;
        wa[0] = (uint8_t)(int8_t)q0; wa[2] = (uint8_t)(int8_t)q1;
        wb[0] = (uint8_t)(int8_t)q2; wb[2] = (uint8_t)(int8_t)q3;
        if (sub == 0) {
            const float dq = __half2float(__float2half_rn(d));
            dxs[b] = dq;
            dx8[b] = dq * 8.f * (float)qsum;
        }
    }
}

// Integer dot product of one quant block: the 32 nibbles in q against the block's q80 planes A and B. High nibbles are used
// in place (q & 0xf0f0f0f0 = 16 * nibble); one shift removes the factor 16, exactly, since their partial sum is a multiple of 16.
__device__ __forceinline__ int q40q80Dot(const uint4 &q, const uint4 &A, const uint4 &B) {
    const uint32_t ml = 0x0f0f0f0fu, mh = 0xf0f0f0f0u;
    int lo = dp4a(q.x & ml, A.x, 0), hi = dp4a(q.x & mh, B.x, 0);
    lo = dp4a(q.y & ml, A.y, lo); hi = dp4a(q.y & mh, B.y, hi);
    lo = dp4a(q.z & ml, A.z, lo); hi = dp4a(q.z & mh, B.z, hi);
    lo = dp4a(q.w & ml, A.w, lo); hi = dp4a(q.w & mh, B.w, hi);
    return lo + (hi >> 4);
}

// One step of a ring stage: the lane's quant block blk of the 4 stage rows rl..rl+3 (sq / ss: the stage's nibbles and scales,
// nblk blocks a row) against NB activation vectors (token t at planeA / planeB / dxs / dx8 + t * nblk).
// acc[r][t] = d_w * (d_x * dot - 8 * d_x * sum(q)), 0 for lanes past the row.
template <int NB>
__device__ __forceinline__ void stageStepDot(const uint4 *sq, const uint16_t *ss, uint32_t rl, uint32_t blk, uint32_t nblk,
                                             const uint4 *planeA, const uint4 *planeB, const float *dxs, const float *dx8,
                                             float (&acc)[kRowsPerStep][NB]) {
#pragma unroll
    for (int r = 0; r < kRowsPerStep; r++)
#pragma unroll
        for (int t = 0; t < NB; t++) acc[r][t] = 0.f;
    if (blk >= nblk) return;
    uint4 A[NB], B[NB];
    float dxv[NB], dx8v[NB];
#pragma unroll
    for (int t = 0; t < NB; t++) {
        A[t] = planeA[t * nblk + blk];
        B[t] = planeB[t * nblk + blk];
        dxv[t] = dxs[t * nblk + blk];
        dx8v[t] = dx8[t * nblk + blk];
    }
    // Rows past the end of a short last stage read stale ring bytes (always inside the stage buffer because stageRows % 4 == 0);
    // the callers do not store their sums.
    const uint4 *qp = sq + rl * nblk + blk;
    const uint16_t *sp = ss + rl * nblk + blk;
#pragma unroll
    for (int r = 0; r < kRowsPerStep; r++) {
        const uint4 q = qp[r * nblk];
        const float dw = __half2float(__ushort_as_half(sp[r * nblk]));
#pragma unroll
        for (int t = 0; t < NB; t++) acc[r][t] = dw * (dxv[t] * (float)q40q80Dot(q, A[t], B[t]) - dx8v[t]);
    }
}

// Row r's output for token t: its per-segment partials ([rows][nseg][NB]) summed in segment order.
template <int NB>
__device__ __forceinline__ float segRowSum(const float *partial, uint32_t r, uint32_t t, uint32_t nseg) {
    float v = 0.f;
    for (uint32_t sg = 0; sg < nseg; sg++) v += partial[((size_t)r * nseg + sg) * NB + t];
    return v;
}

// ---- greedy arg-max over the logits rows of a grid: the lowest index among equal maxima wins ----
__device__ __forceinline__ void argMaxMerge(float &best, int &bestIdx, float v, int i) {
    if (v > best || (v == best && i < bestIdx)) { best = v; bestIdx = i; }
}
__device__ __forceinline__ void warpArgMax(float &best, int &bestIdx) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bestIdx, o);
        argMaxMerge(best, bestIdx, ov, oi);
    }
}

struct ArgMaxOut {
    float *val;              // [grid] per-CTA best value
    int *idx;                // [grid] per-CTA best index
    unsigned int *counter;   // zero-initialised, self-resetting
    int *token;              // the winning index (null: the token, position and history are not written)
    int *pos, *history;      // pos[0] += 1, then history[pos] = token while pos < historyCap (history may be null)
    uint32_t historyCap;
};

// Consumer warps of a TMA-fed GEMV, after each thread has reduced its rows to (best, bestIdx): the CTA's candidate goes to
// o.val / o.idx, and the last CTA to arrive reduces all candidates. Under tensor parallelism (ar.nRanks > 1) the ranks'
// winners are exchanged over the LL candidate words, so every rank picks the same global token. stop() is called once per
// poll of a peer's word; true ends the wait. `red` holds 32 floats of shared memory.
template <typename Stop>
__device__ __forceinline__ void argMaxEpilogue(float best, int bestIdx, float *red, const ArgMaxOut &o, const ArArgs &ar, int tid,
                                               Stop stop) {
    const int lane = tid & 31, warp = tid >> 5;
    warpArgMax(best, bestIdx);
    float *sv = red;                                   // 16 floats
    int *si = reinterpret_cast<int *>(red + 16);
    consumerBarrier();
    if (lane == 0) { sv[warp] = best; si[warp] = bestIdx; }
    consumerBarrier();
    __shared__ bool lastCta;
    if (warp == 0) {
        best = lane < kConsumerWarps ? sv[lane] : -INFINITY;
        bestIdx = lane < kConsumerWarps ? si[lane] : 0x7fffffff;
        warpArgMax(best, bestIdx);
        if (lane == 0) {
            o.val[blockIdx.x] = best;
            o.idx[blockIdx.x] = bestIdx;
            __threadfence();
            const unsigned int prev = atomicAdd(o.counter, 1u);
            lastCta = prev == gridDim.x - 1;
            if (lastCta) *o.counter = 0;
        }
    }
    consumerBarrier();
    if (!lastCta || warp != 0) return;
    __threadfence();
    best = -INFINITY;
    bestIdx = 0x7fffffff;
    for (uint32_t i = lane; i < gridDim.x; i += 32) argMaxMerge(best, bestIdx, __ldcg(o.val + i), __ldcg(o.idx + i));
    warpArgMax(best, bestIdx);
    if (ar.nRanks > 1) {
        if (lane < ar.nRanks) stLL(ar.cand[lane] + ar.rank, __float_as_uint(best), (uint32_t)bestIdx + 1u);
        if (lane < ar.nRanks) {
            uint64_t *w = ar.cand[ar.rank] + lane;
            uint2 v = ldLL(w);
            while (v.y == 0u && !stop()) v = ldLL(w);
            best = __uint_as_float(v.x);
            bestIdx = (int)(v.y - 1u);
            stLL(w, 0u, 0u);
        } else {
            best = -INFINITY;
            bestIdx = 0x7fffffff;
        }
        warpArgMax(best, bestIdx);
    }
    if (lane == 0 && o.token) {
        o.token[0] = bestIdx;
        const int p = o.pos[0] + 1;
        o.pos[0] = p;
        if (o.history && (uint32_t)p < o.historyCap) o.history[p] = bestIdx;
    }
}

// Per-row arg-max of an NB-row logits launch (NB > 1, one rank): every consumer thread has reduced its rows of logits row
// tid % NB to (best, bestIdx). Each CTA leaves row t's candidate at o.val / o.idx [t * grid + cta]; the last CTA to arrive
// writes row t's winner, the lowest index among equal maxima, to o.token[t]. Positions and history are not touched.
// `scratch` holds 2 * kConsumerWarps * NB words of shared memory that no consumer reads any more.
template <int NB>
__device__ __forceinline__ void argMaxRowsEpilogue(float best, int bestIdx, float *scratch, const ArgMaxOut &o, int tid) {
    static_assert(NB > 1 && NB <= 8 && (NB & (NB - 1)) == 0, "rows of a batched launch");
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int off = 16; off >= NB; off >>= 1) {   // lanes with the same lane % NB hold the same row
        const float ov = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bestIdx, off);
        argMaxMerge(best, bestIdx, ov, oi);
    }
    float *sv = scratch;
    int *si = reinterpret_cast<int *>(scratch + kConsumerWarps * NB);
    consumerBarrier();
    if (lane < NB) { sv[warp * NB + lane] = best; si[warp * NB + lane] = bestIdx; }
    consumerBarrier();
    __shared__ bool lastCta;
    if (warp == 0) {
        if (lane < NB) {
            best = -INFINITY;
            bestIdx = 0x7fffffff;
            for (int w = 0; w < kConsumerWarps; w++) argMaxMerge(best, bestIdx, sv[w * NB + lane], si[w * NB + lane]);
            o.val[lane * gridDim.x + blockIdx.x] = best;
            o.idx[lane * gridDim.x + blockIdx.x] = bestIdx;
            __threadfence();
        }
        __syncwarp();
        if (lane == 0) {
            const unsigned int prev = atomicAdd(o.counter, 1u);
            lastCta = prev == gridDim.x - 1;
            if (lastCta) *o.counter = 0;
        }
    }
    consumerBarrier();
    if (!lastCta || warp >= NB) return;
    __threadfence();
    best = -INFINITY;
    bestIdx = 0x7fffffff;
    for (uint32_t i = lane; i < gridDim.x; i += 32)
        argMaxMerge(best, bestIdx, __ldcg(o.val + warp * gridDim.x + i), __ldcg(o.idx + warp * gridDim.x + i));
    warpArgMax(best, bestIdx);
    if (lane == 0) o.token[warp] = bestIdx;
}

}  // namespace dl
