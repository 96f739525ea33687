// Per-token log-probabilities for the chat APIs' `logprobs` / `top_logprobs` (kernels.h: launchLogprobsRows).
//
// One CTA per row, rows read straight from the device logits: nothing crosses PCIe but the small result block.
// - Pass 1 reads the row once. Every thread keeps an online (max, sum of exp) pair over a strided share of the row: exp through
//   expNeg (dl_expf.h), the sum in double, rescaled in double when the thread's max rises. The pairs combine by a fixed tree,
//   so the numbers are bitwise reproducible and do not depend on the other rows of a launch.
// - Top k without sorting the vocabulary: the k-th largest of the 32 warp maxima is a lower bound t0 of the row's k-th largest
//   value (k distinct entries reach it). Pass 2 collects every entry whose key reaches t0 (usually a few dozen) and ranks them
//   by (value desc, id asc). When more than kCand entries reach t0 (many ties near the top, a flat row), a radix descent over
//   the keys (8 bits a level, integer histograms: order independent, as the sampler's) finds the exact key T of the k-th
//   largest, and a last pass in index order takes the entries above T plus the lowest ids holding T.
#include "../common/dl_expf.h"
#include "kernels.h"

namespace dl {
namespace {

constexpr int kLpThreads = 1024;
constexpr int kCand = kLpThreads;   // candidate buffer of the fast path
constexpr int kUnroll = 8;          // loads in flight per thread in the passes over the row

struct LpArgs {
    const float *logits;
    uint32_t logitsStride, n, rowMask;
    const int *chosen;
    int32_t *out;
    SampleControls ctl;
    const float *rowParams;
    uint8_t k[32];
};

// Order-preserving key: a larger value has a larger key; -0 and +0 share one.
__device__ __forceinline__ uint32_t orderKey(float v) {
    const uint32_t u = __float_as_uint(__fadd_rn(v, 0.0f));
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ double warpSumD(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ uint32_t warpMaxU(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Exclusive prefix of v over the block in thread order.
__device__ uint32_t blockExclusiveScanU(uint32_t v, uint32_t *warpTotals) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) warpTotals[warp] = inc;
    __syncthreads();
    const uint32_t wt = warpTotals[lane];
    uint32_t winc = wt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
    }
    return __shfl_sync(0xffffffffu, winc - wt, warp) + inc - v;
}

struct LpRow {
    const float *x;
    SampleControls c;
    bool ctl;
    int chosen;
    __device__ __forceinline__ float value(uint32_t i) const { return ctl ? controlled(c, x[i], i, chosen) : x[i]; }
};

__device__ __forceinline__ int32_t logprobBits(float v, double lse) { return __float_as_int(__double2float_rn((double)v - lse)); }

__global__ void __launch_bounds__(kLpThreads, 1) logprobsRowsKernel(LpArgs a) {
    __shared__ double redD[32];
    __shared__ float redF[32];
    __shared__ uint32_t redU[32];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t candKey[kCand];
    __shared__ int candId[kCand];
    __shared__ uint32_t sCount, sKey, sAbove;
    const uint32_t row = blockIdx.x;
    if (!((a.rowMask >> row) & 1u)) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n = a.n;
    LpRow r;
    r.x = a.logits + (size_t)row * a.logitsStride;
    r.c = a.ctl;
    r.ctl = r.c.bias || r.c.counts;
    if (r.c.counts) r.c.counts += (size_t)row * r.c.countsStride;
    if (r.c.bias) r.c.bias += (size_t)row * r.c.biasStride;
    if (a.rowParams) { r.c.presence = a.rowParams[4 * row + 2]; r.c.frequency = a.rowParams[4 * row + 3]; }
    r.chosen = a.chosen[row];
    const int k = min((int)a.k[row], min(kLogprobsMaxTop, (int)n));
    int32_t *out = a.out + (size_t)row * kLogprobsWords;

    // pass 1: online max and sum of exp per thread, over ids threadIdx.x + j * kLpThreads in increasing order; kUnroll loads are
    // issued before any is used, or the loop waits out one memory latency per entry
    float m = -INFINITY;
    double s = 0.0;
    for (uint32_t i0 = threadIdx.x; i0 < n; i0 += kUnroll * kLpThreads) {
        float v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const uint32_t i = i0 + u * kLpThreads;
            v[u] = i < n ? r.value(i) : -INFINITY;   // -inf adds expNeg(-inf) = +0
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            if (v[u] > m) { s *= exp((double)m - (double)v[u]); m = v[u]; }
            s += (double)expNeg(__fsub_rn(v[u], m));
        }
    }
    float M = warpMax(m);
    const uint32_t warpTop = warpMaxU(m == -INFINITY ? 0u : orderKey(m));
    if (lane == 0) { redF[warp] = M; redU[warp] = warpTop; }
    __syncthreads();
    M = warpMax(redF[lane]);
    double S = warpSumD(m == -INFINITY ? 0.0 : s * exp((double)m - (double)M));
    if (lane == 0) redD[warp] = S;
    __syncthreads();
    S = warpSumD(redD[lane]);
    const double lse = (double)M + log(S);
    if (threadIdx.x == 0) {
        out[0] = r.chosen;
        out[1] = (r.chosen >= 0 && (uint32_t)r.chosen < n) ? logprobBits(r.value(r.chosen), lse) : 0x7fc00000;
        out[2] = k;
        out[3] = 0;
    }
    for (int w = 4 + 2 * k + threadIdx.x; w < kLogprobsWords; w += kLpThreads) out[w] = 0;
    if (k == 0) return;

    // t0: the k-th largest warp maximum (key 0: a warp that saw no entry; then every entry is a candidate)
    if (warp == 0) {
        const uint32_t mine = redU[lane];
        int rank = 0;
        for (int j = 0; j < 32; j++) {
            const uint32_t o = __shfl_sync(0xffffffffu, mine, j);
            rank += (o > mine || (o == mine && j < lane)) ? 1 : 0;
        }
        if (rank == k - 1) sKey = mine;
        if (lane == 0) sCount = 0;
    }
    __syncthreads();
    const uint32_t t0 = sKey;

    // pass 2: every entry whose key reaches t0 (uniform trip count: whole warps vote)
    for (uint32_t i0 = 0; i0 < n; i0 += kUnroll * kLpThreads) {
        uint32_t key[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const uint32_t i = i0 + u * kLpThreads + threadIdx.x;
            key[u] = i < n ? orderKey(r.value(i)) : 0u;
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const uint32_t i = i0 + u * kLpThreads + threadIdx.x;
            const bool take = i < n && key[u] >= t0;
            const uint32_t votes = __ballot_sync(0xffffffffu, take);
            uint32_t base = 0;
            if (lane == 0 && votes) base = atomicAdd(&sCount, (uint32_t)__popc(votes));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (take) {
                const uint32_t slot = base + __popc(votes & ((1u << lane) - 1u));
                if (slot < (uint32_t)kCand) { candKey[slot] = key[u]; candId[slot] = (int)i; }
            }
        }
    }
    __syncthreads();
    uint32_t nCand = sCount;
    if (nCand > (uint32_t)kCand) {
        // radix descent to the exact key T of the k-th largest entry; sAbove counts the entries above the decided prefix range
        uint32_t prefix = 0, above = 0;
        for (int level = 0; level < 4; level++) {
            const int shift = 24 - 8 * level;
            for (int b = threadIdx.x; b < 256; b += kLpThreads) hist[b] = 0;
            __syncthreads();
            for (uint32_t i0 = 0; i0 < n; i0 += kLpThreads) {
                const uint32_t i = i0 + threadIdx.x;
                uint32_t bin = 256;
                if (i < n) {
                    const uint32_t key = orderKey(r.value(i));
                    if (level == 0 || (key >> (shift + 8)) == prefix) bin = (key >> shift) & 255u;
                }
                const uint32_t peers = __match_any_sync(0xffffffffu, bin);
                if (bin < 256 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
            }
            __syncthreads();
            if (warp == 0) {   // lane l holds bins 8l .. 8l + 7; find the bin where the count from the top reaches k
                uint32_t tot = 0;
                for (int b = 0; b < 8; b++) tot += hist[8 * lane + b];
                uint32_t suf = tot;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t t = __shfl_down_sync(0xffffffffu, suf, o);
                    if (lane + o < 32) suf += t;
                }
                uint32_t run = above + suf - tot;
                if (run < (uint32_t)k && (uint32_t)k <= run + tot) {
                    for (int b = 7; b >= 0; b--) {
                        const uint32_t h = hist[8 * lane + b];
                        if (run + h >= (uint32_t)k) { sKey = 8 * lane + b; sAbove = run; break; }
                        run += h;
                    }
                }
            }
            __syncthreads();
            prefix = (prefix << 8) | sKey;
            above = sAbove;
            __syncthreads();
        }
        // entries above T (fewer than k) and the lowest ids holding T, k in all
        const uint32_t need = (uint32_t)k - above;
        const uint32_t chunk = (n + kLpThreads - 1) / kLpThreads;
        const uint32_t lo = min(threadIdx.x * chunk, n), hi = min(lo + chunk, n);
        uint32_t ties = 0;
        for (uint32_t i = lo; i < hi; i++) ties += orderKey(r.value(i)) == prefix ? 1u : 0u;
        uint32_t before = blockExclusiveScanU(ties, redU);
        if (threadIdx.x == 0) sCount = 0;
        __syncthreads();
        for (uint32_t i = lo; i < hi; i++) {
            const uint32_t key = orderKey(r.value(i));
            bool take = key > prefix;
            if (key == prefix) take = before++ < need;
            if (take) {
                const uint32_t slot = atomicAdd(&sCount, 1u);
                candKey[slot] = key;
                candId[slot] = (int)i;
            }
        }
        __syncthreads();
        nCand = sCount;
    }

    // rank the candidates by (value desc, id asc); the first k are the answer
    for (uint32_t j = threadIdx.x; j < nCand; j += kLpThreads) {
        const uint32_t kj = candKey[j];
        const int ij = candId[j];
        uint32_t rank = 0;
        for (uint32_t q = 0; q < nCand && rank < (uint32_t)k; q++) {
            const uint32_t kq = candKey[q];
            rank += (kq > kj || (kq == kj && candId[q] < ij)) ? 1u : 0u;
        }
        if (rank < (uint32_t)k) {
            out[4 + 2 * rank] = ij;
            out[5 + 2 * rank] = logprobBits(r.value(ij), lse);
        }
    }
}

}  // namespace

int launchLogprobsRows(const float *logits, uint32_t logitsStride, uint32_t n, uint32_t B, uint32_t rowMask, const int *k, const int *chosen,
                       int32_t *out, cudaStream_t stream, const SampleControls *controls, const float *rowParams) {
    if (n < 1 || B < 1 || B > 32) return -1;
    LpArgs a{};
    a.logits = logits; a.logitsStride = logitsStride; a.n = n; a.chosen = chosen; a.out = out; a.rowParams = rowParams;
    a.rowMask = B == 32 ? rowMask : rowMask & ((1u << B) - 1u);
    for (uint32_t b = 0; b < B; b++) {
        if (k[b] < 0 || k[b] > kLogprobsMaxTop) return -2;
        a.k[b] = (uint8_t)k[b];
    }
    if (controls) a.ctl = *controls;
    if (a.rowMask == 0) return 0;
    logprobsRowsKernel<<<B, kLpThreads, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace dl

// Stand-alone entry for tests: log-probabilities of B rows (device f32, row b at logits + b * logitsStride, 0: one row for all) over
// the first n ids; k (host [B], 0..20) top entries per row; chosen (device [B]) the token each row drew; rows outside rowMask read
// nothing. Controls as dl_sample_rows_per_row (bias, counts and rowParams may be null; without rowParams every row takes presence
// and frequency); counts are those after the draw of chosen[b]. out: device int32 [B][kLogprobsWords] (kernels.h).
DL_EXPORT int dl_logprobs_rows(const float *logits, uint32_t logitsStride, uint32_t n, uint32_t B, uint32_t rowMask, const int *k, const int *chosen,
                               const float *bias, uint32_t biasStride, uint32_t *counts, uint32_t countsStride, float presence, float frequency,
                               const float *rowParams, int32_t *out, cudaStream_t stream) {
    const dl::SampleControls ctl{bias, counts, countsStride, presence, frequency, biasStride};
    return dl::launchLogprobsRows(logits, logitsStride, n, B, rowMask, k, chosen, out, stream, (bias || counts) ? &ctl : nullptr, rowParams);
}
