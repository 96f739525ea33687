// Temperature / top-p sampling on the device: the logits never leave the GPU.
//
// Semantics = the reference's Sampler::sample (src/tokenizer.cpp:426-512; host twin: csrc/host/text.cpp Sampler::sample):
//   logits / T -> softmax -> coin = xorshift* F32 -> multinomial CDF walk (topp outside (0,1)) or nucleus sampling: drop
//   probabilities below (1 - topp) / (n - 1), order the rest by (probability desc, index asc), cut at the first prefix whose sum
//   exceeds topp, draw r = coin * prefix sum and walk the order until the running sum exceeds r.
// No sort is materialised: both "first prefix whose sum exceeds X" questions are answered by a radix descent over the float keys
// (4 levels x 8 bits, a 256-bin histogram of probability mass per level) followed by a rank selection among equal keys. All
// prefix arithmetic is 2^-40 fixed point in 64-bit integers, so histogram atomics are order independent: the sampler is bit
// reproducible run to run and across ranks — under tensor parallelism every rank samples the same token from the gathered
// logits with its own copy of the generator state, and no token broadcast is needed.
// The filters top_k / min_p (kernels.h: SampleFilters) zero every id outside the candidate set before the normaliser; top_k finds
// its threshold by the same radix descent over counts instead of mass (topKFilter).
//
// Tensor parallelism (K4, reference: gather of vocab slices to the root, src/llm.cpp:587-599): logitsGatherKernel pushes this
// rank's vocabulary slice into every rank's gather buffer (one multimem.st per 16 bytes through the NVSwitch multicast mapping, or
// unicast peer stores) and bumps an arrival counter on every rank; the sampler waits for nRanks arrivals. No NCCL on the step path.
#include "../common/dl_expf.h"
#include "kernels.h"

namespace dl {
namespace {

constexpr int kSampThreads = 1024;
constexpr float kFix = 1099511627776.0f;   // 2^40

__device__ __forceinline__ unsigned long long toFix(float p) { return (unsigned long long)(p * kFix); }

struct SampleArgs {
    const float *logits;       // [n] (full vocabulary on this rank: local buffer or the gather buffer)
    float *probs;              // [n] scratch: exp((l - max) / T)
    uint32_t n;
    float temperature, topp;
    unsigned long long *rng;   // xorshift* state
    int *tokenOut, *pos, *history;
    uint32_t historyCap;
    // tensor parallelism: wait until every rank's slice has arrived in `logits`
    const unsigned int *gatherFlag;
    unsigned int *gatherEpoch;     // device counter of completed gathers (the kernel advances it)
    uint32_t nRanks;
    int *debugOut;             // optional [4]: {last index in order?, ...} unused by the product path
    // batched draws (grid B, one CTA per row): row b reads logits + b * logitsStride, probs + b * probsStride, rng[b], tokenOut[b]
    uint32_t logitsStride, probsStride, inactiveMask;
    SampleControls ctl;        // bias / penalties (kernels.h); row b counts at ctl.counts + b * ctl.countsStride
    const float *rowParams;    // [B][4] per-row {temperature, top-p, presence, frequency}, or null (launchSampleRows)
    uint32_t topK;             // filters (kernels.h: SampleFilters); 0 / 0.f: off
    float minP;
    const SampleFilters *rowFilters;   // [B] per-row filters in place of topK / minP, or null
};

__device__ float blockMax(float v, float *red) {
    v = warpMax(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = red[lane];          // 32 warps
    t = warpMax(t);
    return t;
}

// Deterministic block sum: fixed tree over warps.
__device__ float blockSum(float v, float *red) {
    v = warpSum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = red[lane];
    t = warpSum(t);
    return t;
}

// Exclusive prefix over the 1024 threads (thread order), for 64-bit integers; returns the exclusive prefix, *total gets the sum.
__device__ unsigned long long blockExclusiveScan(unsigned long long v, unsigned long long *warpTotals, unsigned long long *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) warpTotals[warp] = inc;
    __syncthreads();
    unsigned long long wt = warpTotals[lane];
    unsigned long long winc = wt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
    }
    const unsigned long long warpExcl = __shfl_sync(0xffffffffu, winc - wt, warp);
    if (total) *total = __shfl_sync(0xffffffffu, winc, 31);
    return warpExcl + inc - v;
}

// Finds, in the order (key desc, index asc) over the candidates (prob >= cutoff), the first element whose inclusive prefix sum
// (fixed point) exceeds `target`. Outputs its index and that prefix sum. If the total candidate mass does not exceed the target,
// returns the LAST element of the order and the total (the reference's loop falls off its end the same way).
struct Found { int index; unsigned long long prefix; };

__device__ Found radixFind(const SampleArgs &a, float inv, float cutoff, unsigned long long target, unsigned long long *hist /*[256]*/,
                           unsigned long long *scratch /*[64]*/, int *sInt /*[8]*/) {
    const uint32_t n = a.n;
    uint32_t prefix = 0;                 // decided high bits of the key
    unsigned long long base = 0;         // mass of all candidates whose key is above the current prefix range
    bool exhausted = false;              // the whole candidate mass is <= target
    for (int level = 0; level < 4; level++) {
        const int shift = 24 - 8 * level;
        for (int b = threadIdx.x; b < 256; b += kSampThreads) hist[b] = 0;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += kSampThreads) {
            const float p = a.probs[i] * inv;
            if (p < cutoff) continue;
            const uint32_t key = __float_as_uint(p);
            if (level > 0 && (key >> (shift + 8)) != prefix) continue;
            atomicAdd(&hist[(key >> shift) & 255u], toFix(p));
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long run = base;
            int chosen = -1, lowestNonEmpty = -1;
            for (int b = 255; b >= 0; b--) {
                if (hist[b] == 0) continue;
                lowestNonEmpty = b;
                if (run + hist[b] > target) { chosen = b; break; }
                run += hist[b];
            }
            if (chosen < 0) {            // never exceeds: continue towards the smallest key so that the last element is found
                chosen = lowestNonEmpty;
                run -= (lowestNonEmpty >= 0 ? hist[lowestNonEmpty] : 0);
                sInt[1] = 1;
            } else {
                sInt[1] = 0;
            }
            sInt[0] = chosen;
            scratch[0] = run;
        }
        __syncthreads();
        if (sInt[0] < 0) return Found{(int)n - 1, base};     // no candidate at all (cannot happen for n >= 2: max prob >= 1/n > cutoff)
        exhausted = exhausted || sInt[1] != 0;
        prefix = (prefix << 8) | (uint32_t)sInt[0];
        base = scratch[0];
        __syncthreads();
    }
    // all elements with key == prefix share one probability p*: pick the j-th in index order
    const float pStar = __uint_as_float(prefix);
    const unsigned long long fStar = toFix(pStar);
    // per-thread contiguous index chunks keep the index order
    const uint32_t chunk = (n + kSampThreads - 1) / kSampThreads;
    const uint32_t lo = threadIdx.x * chunk, hi = min(lo + chunk, n);
    unsigned long long cnt = 0;
    for (uint32_t i = lo; i < hi; i++) cnt += (__float_as_uint(a.probs[i] * inv) == prefix) ? 1ull : 0ull;
    unsigned long long totalTies = 0;
    const unsigned long long before = blockExclusiveScan(cnt, scratch + 8, &totalTies);
    // number of ties needed: smallest j >= 1 with base + j * f* > target (all of them when the mass is exhausted)
    unsigned long long need;
    if (exhausted || base + totalTies * fStar <= target) need = totalTies;
    else need = (target - base) / fStar + 1;       // base <= target here
    if (need < 1) need = 1;
    if (need > totalTies) need = totalTies;
    __syncthreads();
    if (before < need && need <= before + cnt) {
        unsigned long long seen = before;
        for (uint32_t i = lo; i < hi; i++) {
            if (__float_as_uint(a.probs[i] * inv) == prefix && ++seen == need) { sInt[2] = (int)i; break; }
        }
    }
    __syncthreads();
    return Found{sInt[2], base + need * fStar};
}

// top_k filter over the unnormalised probabilities in a.probs (a.topK < number of nonzero-or-kept ids): finds the K-th key in
// the order (key desc, index asc) by a radix descent over counts (4 levels x 8 bits, a 256-bin u32 histogram per level; the keys
// are non-negative floats, so their bit patterns order like their values), then keeps every key above it and the lowest-index ties
// up to K in all. Zeroes every other id; returns this thread's fixed-point sum over its contiguous index chunk of the kept ones.
__device__ unsigned long long topKFilter(const SampleArgs &a, unsigned long long *histMem, unsigned long long *scratch, int *sInt) {
    const uint32_t n = a.n, K = a.topK;
    unsigned int *hist = reinterpret_cast<unsigned int *>(histMem);
    const int lane = threadIdx.x & 31;
    uint32_t prefix = 0;   // decided high bits of the K-th key
    uint32_t above = 0;    // ids whose key is above the current prefix range
    for (int level = 0; level < 4; level++) {
        const int shift = 24 - 8 * level;
        for (int b = threadIdx.x; b < 256; b += kSampThreads) hist[b] = 0;
        __syncthreads();
        // every thread runs the same trip count, so whole warps aggregate equal bins before the shared atomic
        for (uint32_t base = 0; base < n; base += kSampThreads) {
            const uint32_t i = base + threadIdx.x;
            uint32_t bin = 256u;
            if (i < n) {
                const uint32_t key = __float_as_uint(a.probs[i]);
                if (level == 0 || (key >> (shift + 8)) == prefix) bin = (key >> shift) & 255u;
            }
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (bin < 256u && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned)__popc(peers));
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t run = above;
            int chosen = 0;
            for (int b = 255; b >= 0; b--) {
                if (run + hist[b] >= K) { chosen = b; break; }
                run += hist[b];
            }
            sInt[0] = chosen;
            sInt[1] = (int)run;
        }
        __syncthreads();
        prefix = (prefix << 8) | (uint32_t)sInt[0];
        above = (uint32_t)sInt[1];
        __syncthreads();
    }
    // keep the K - above lowest indices among the keys equal to the K-th key (per-thread contiguous chunks keep the index order)
    const uint32_t chunk = (n + kSampThreads - 1) / kSampThreads;
    const uint32_t lo = threadIdx.x * chunk, hi = min(lo + chunk, n);
    unsigned long long ties = 0;
    for (uint32_t i = lo; i < hi; i++) ties += (__float_as_uint(a.probs[i]) == prefix) ? 1ull : 0ull;
    unsigned long long seen = blockExclusiveScan(ties, scratch + 8, nullptr);
    const unsigned long long need = K - above;
    unsigned long long sFix = 0;
    for (uint32_t i = lo; i < hi; i++) {
        const float e = a.probs[i];
        const uint32_t key = __float_as_uint(e);
        if (key > prefix || (key == prefix && seen++ < need)) sFix += toFix(e);
        else a.probs[i] = 0.f;
    }
    return sFix;
}

// Temperature / top-p draw from src (logits, or the transformed logits under controls) whose maximum after division by T is m.
// Filtered: the row's top_k / min_p (kernels.h: SampleFilters) are active; the unfiltered instance is the draw without them.
template <bool Filtered>
__device__ int drawSampled(const SampleArgs &a, const float *src, float m, unsigned long long *hist, unsigned long long *scratch, int *sInt,
                           float *sCoin) {
    const uint32_t n = a.n;
    // per-thread sums over contiguous chunks (index order), combined by a fixed tree
    const uint32_t chunk = (n + kSampThreads - 1) / kSampThreads;
    const uint32_t lo = threadIdx.x * chunk, hi = min(lo + chunk, n);
    // min_p threshold: max e = expNeg(max(x / T) - m) = expNeg(m - m) (1 for a finite maximum, 0 otherwise)
    const bool useMinP = Filtered && a.minP > 0.f;
    const float eMax = Filtered ? expNeg(__fsub_rn(m, m)) : 0.f;
    const float thr = useMinP ? __fmul_rn(a.minP, eMax) : 0.f;
    unsigned long long sFix = 0, kept = 0;
    for (uint32_t i = lo; i < hi; i++) {
        float e = expNeg(__fsub_rn(__fdiv_rn(src[i], a.temperature), m));
        if (useMinP) {
            if (e < thr) e = 0.f;
            else kept++;
        }
        a.probs[i] = e;
        sFix += toFix(e);
    }
    unsigned long long nS = n;   // |S|: ids in the candidate set
    if (Filtered) {
        if (useMinP) (void)blockExclusiveScan(kept, scratch + 8, &nS);
        if (a.topK && a.topK < nS) {
            __syncthreads();
            sFix = topKFilter(a, hist, scratch, sInt);
            nS = a.topK;
        }
    }
    unsigned long long sTotal = 0;
    (void)blockExclusiveScan(sFix, scratch + 8, &sTotal);
    const float inv = __fdiv_rn(1.0f, __fdiv_rn((float)sTotal, kFix));
    if (threadIdx.x == 0) {
        unsigned long long st = *a.rng;          // xorshift* (reference src/tokenizer.cpp:25-36)
        st ^= st >> 12; st ^= st << 25; st ^= st >> 27;
        *a.rng = st;
        const uint32_t u = (uint32_t)((st * 0x2545F4914F6CDD1Dull) >> 32);
        *sCoin = (float)(u >> 8) * 5.9604644775390625e-8f;   // / 2^24, exact
        sInt[2] = (int)n - 1;
        if (Filtered) sInt[3] = (int)n - 1;
    }
    __syncthreads();
    if (Filtered && nS == 1) {   // one candidate: the id holding max e (the coin is drawn all the same)
        for (uint32_t i = threadIdx.x; i < n; i += kSampThreads) {
            if (a.probs[i] == eMax) { atomicMin(&sInt[3], (int)i); break; }
        }
        __syncthreads();
        return sInt[3];
    }
    const float coin = *sCoin;
    if (a.topp <= 0.f || a.topp >= 1.f) {
        // multinomial walk in index order
        unsigned long long mine = 0;
        for (uint32_t i = lo; i < hi; i++) mine += toFix(a.probs[i] * inv);
        unsigned long long total = 0;
        const unsigned long long before = blockExclusiveScan(mine, scratch + 8, &total);
        const unsigned long long c = toFix(coin);
        if (before <= c && c < before + mine) {
            unsigned long long cdf = before;
            for (uint32_t i = lo; i < hi; i++) {
                cdf += toFix(a.probs[i] * inv);
                if (c < cdf) { sInt[2] = (int)i; break; }
            }
        }
        __syncthreads();
        return sInt[2];
    }
    const float cutoff = __fdiv_rn(1.0f - a.topp, (float)((Filtered ? (uint32_t)nS : n) - 1));
    const Found cut = radixFind(a, inv, cutoff, toFix(a.topp), hist, scratch, sInt);
    // r = coin * cumulative (the reference multiplies the float prefix sum)
    const float cumulative = __fdiv_rn((float)cut.prefix, kFix);
    const unsigned long long r = toFix(coin * cumulative);
    __syncthreads();
    return radixFind(a, inv, cutoff, r, hist, scratch, sInt).index;
}

__global__ void __launch_bounds__(kSampThreads, 1) sampleKernel(SampleArgs a) {
    __shared__ float red[32];
    __shared__ unsigned long long hist[256];
    __shared__ unsigned long long scratch[64];
    __shared__ int sInt[8];
    __shared__ float sCoin;
    const uint32_t n = a.n;
    const uint32_t row = blockIdx.x;
    if (row < 32 && ((a.inactiveMask >> row) & 1u)) return;
    a.logits += (size_t)row * a.logitsStride;
    a.probs += (size_t)row * a.probsStride;
    a.rng += row;
    a.tokenOut += row;
    if (a.ctl.counts) a.ctl.counts += (size_t)row * a.ctl.countsStride;
    if (a.ctl.bias) a.ctl.bias += (size_t)row * a.ctl.biasStride;
    if (a.rowParams) {
        const float *rp = a.rowParams + 4 * (size_t)row;
        a.temperature = rp[0]; a.topp = rp[1]; a.ctl.presence = rp[2]; a.ctl.frequency = rp[3];
    }
    if (a.rowFilters) { a.topK = a.rowFilters[row].topK; a.minP = a.rowFilters[row].minP; }
    if (a.gatherFlag && a.nRanks > 1) {
        if (threadIdx.x == 0) {
            const unsigned int want = (*a.gatherEpoch + 1u) * a.nRanks;
            unsigned int v;
            uint32_t spins = 0;
            do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.gatherFlag) : "memory"); } while ((int)(v - want) < 0 && ++spins < (1u << 28));
            if (gridDim.x == 1) *a.gatherEpoch += 1u;   // batched draws: epochAdvanceKernel runs after the grid
        }
        __syncthreads();
    }
    // With controls the max pass stores the transformed logits in probs, and the later passes read them from there: counts and
    // bias are read once per logit.
    const bool ctl = a.ctl.bias || a.ctl.counts;
    const bool greedy = a.temperature == 0.f;   // reached with controls or per-row parameters only (the launchers refuse it otherwise)
    const float *src = ctl ? a.probs : a.logits;
    // softmax statistics (IEEE division / shared exp / integer normaliser: the host sampler computes the very same numbers)
    float m = -INFINITY;
    for (uint32_t i = threadIdx.x; i < n; i += kSampThreads) {
        float x = a.logits[i];
        if (ctl) { x = controlled(a.ctl, x, i); a.probs[i] = x; }
        m = fmaxf(m, greedy ? x : __fdiv_rn(x, a.temperature));
    }
    m = blockMax(m, red);
    int token;
    if (greedy) {   // arg-max: the lowest index holding the maximum
        if (threadIdx.x == 0) sInt[3] = (int)n - 1;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += kSampThreads) {
            if (src[i] == m) { atomicMin(&sInt[3], (int)i); break; }
        }
        __syncthreads();
        token = sInt[3];
    } else if ((a.topK && a.topK < n) || a.minP > 0.f) {
        token = drawSampled<true>(a, src, m, hist, scratch, sInt, &sCoin);
    } else {
        token = drawSampled<false>(a, src, m, hist, scratch, sInt, &sCoin);
    }
    if (threadIdx.x == 0) {
        a.tokenOut[0] = token;
        if (a.ctl.counts) a.ctl.counts[token] += 1u;
        if (a.pos) {
            const int p = a.pos[0] + 1;
            a.pos[0] = p;
            if (a.history && (uint32_t)p < a.historyCap) a.history[p] = token;
        }
    }
}

__global__ void epochAdvanceKernel(unsigned int *gatherEpoch) { *gatherEpoch += 1u; }

// Copies this rank's vocabulary slice of `rows` logits rows ([rows][v0], local) into the gather buffer of every rank
// ([rows][nRanks * v0]) and signals its arrival.
__global__ void __launch_bounds__(256) logitsGatherKernel(const float *local, uint32_t v0, uint32_t rank, uint32_t nRanks, float *gatherMc,
                                                           float *const *gatherUc, unsigned int *flagMc, unsigned int *const *flagUc,
                                                           unsigned int *blockCounter, uint32_t rows) {
    const uint32_t nVec = v0 / 4;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nVec * rows; i += gridDim.x * blockDim.x) {
        const float4 v = reinterpret_cast<const float4 *>(local)[i];
        const uint32_t row = i / nVec;
        const size_t off = ((size_t)row * nRanks + rank) * v0 + (size_t)(i - row * nVec) * 4;
        if (gatherMc) {
            asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(gatherMc + off), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
        } else {
            for (uint32_t p = 0; p < nRanks; p++) *reinterpret_cast<float4 *>(gatherUc[p] + off) = v;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(blockCounter, 1u);
        if (prev == gridDim.x - 1) {
            *blockCounter = 0;
            __threadfence_system();
            if (flagMc) asm volatile("multimem.red.release.sys.global.add.u32 [%0], 1;" ::"l"(flagMc) : "memory");
            else for (uint32_t p = 0; p < nRanks; p++) asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(flagUc[p]) : "memory");
        }
    }
}

}  // namespace

bool sampleFiltersValid(const SampleFilters &f) { return f.minP >= 0.f && f.minP <= 1.f; }

int launchSample(const float *logits, float *probs, uint32_t n, float temperature, float topp, unsigned long long *rng, int *tokenOut, int *pos,
                 int *history, uint32_t historyCap, const unsigned int *gatherFlag, unsigned int *gatherEpoch, uint32_t nRanks,
                 cudaStream_t stream, const SampleControls *controls, const SampleFilters *filters) {
    if (n < 2 || !(temperature > 0.f || (temperature == 0.f && controls))) return -1;
    if (filters && !sampleFiltersValid(*filters)) return -2;
    SampleArgs a{};
    a.logits = logits; a.probs = probs; a.n = n; a.temperature = temperature; a.topp = topp; a.rng = rng; a.tokenOut = tokenOut; a.pos = pos;
    a.history = history; a.historyCap = historyCap; a.gatherFlag = gatherFlag; a.gatherEpoch = gatherEpoch; a.nRanks = nRanks;
    if (controls) a.ctl = *controls;
    if (filters) { a.topK = filters->topK; a.minP = filters->minP; }
    sampleKernel<<<1, kSampThreads, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int launchLogitsGather(const float *local, uint32_t v0, uint32_t rank, uint32_t nRanks, float *gatherMc, float *const *gatherUcDev,
                       unsigned int *flagMc, unsigned int *const *flagUcDev, unsigned int *blockCounter, cudaStream_t stream, uint32_t rows) {
    if (v0 % 4 || rows < 1) return -1;
    logitsGatherKernel<<<32, 256, 0, stream>>>(local, v0, rank, nRanks, gatherMc, gatherUcDev, flagMc, flagUcDev, blockCounter, rows);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int launchSampleRows(const float *logits, uint32_t logitsStride, float *probs, uint32_t n, float temperature, float topp, unsigned long long *rng,
                     int *tokenOut, uint32_t B, uint32_t inactiveMask, const unsigned int *gatherFlag, unsigned int *gatherEpoch, uint32_t nRanks,
                     cudaStream_t stream, const SampleControls *controls, const float *rowParams, const SampleFilters *filters,
                     const SampleFilters *rowFilters) {
    if (n < 2 || !(temperature > 0.f || (temperature == 0.f && (controls || rowParams))) || B < 1 || B > 32) return -1;
    if (filters && !sampleFiltersValid(*filters)) return -2;
    SampleArgs a{};
    a.logits = logits; a.probs = probs; a.n = n; a.temperature = temperature; a.topp = topp; a.rng = rng; a.tokenOut = tokenOut;
    a.gatherFlag = gatherFlag; a.gatherEpoch = gatherEpoch; a.nRanks = nRanks;
    a.logitsStride = logitsStride; a.probsStride = n; a.inactiveMask = inactiveMask; a.rowParams = rowParams;
    if (controls) a.ctl = *controls;
    if (filters) { a.topK = filters->topK; a.minP = filters->minP; }
    a.rowFilters = rowFilters;
    sampleKernel<<<B, kSampThreads, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    if (gatherFlag && nRanks > 1 && B > 1) {
        epochAdvanceKernel<<<1, 1, 0, stream>>>(gatherEpoch);
        DL_CUDA_CHECK(cudaGetLastError());
    }
    return 0;
}

}  // namespace dl

// Stand-alone entry for tests: samples one token from `logits` (device f32 [n]); rngState is a device u64.
DL_EXPORT int dl_sample_logits(const float *logits, float *probsScratch, uint32_t n, float temperature, float topp, unsigned long long *rngState,
                               int *tokenOut, cudaStream_t stream) {
    return dl::launchSample(logits, probsScratch, n, temperature, topp, rngState, tokenOut, nullptr, nullptr, 0, nullptr, nullptr, 1, stream);
}

// Stand-alone entry for tests: B draws from logits rows (device f32, row b at logits + b * logitsStride; 0 = all rows from one row),
// with the generators rngState[0..B) (device u64) and B * n floats of scratch.
DL_EXPORT int dl_sample_rows(const float *logits, uint32_t logitsStride, float *probsScratch, uint32_t n, float temperature, float topp,
                             unsigned long long *rngState, int *tokenOut, uint32_t B, uint32_t inactiveMask, cudaStream_t stream) {
    return dl::launchSampleRows(logits, logitsStride, probsScratch, n, temperature, topp, rngState, tokenOut, B, inactiveMask, nullptr, nullptr, 1,
                                stream);
}

// dl_sample_rows with sampling controls (kernels.h: SampleControls): bias (device f32 [n], may be null), counts (device u32, row b at
// counts + b * countsStride, may be null; every draw increments it) and the two penalties. Temperature 0 draws the arg-max.
DL_EXPORT int dl_sample_rows_controlled(const float *logits, uint32_t logitsStride, float *probsScratch, uint32_t n, float temperature, float topp,
                                        unsigned long long *rngState, int *tokenOut, uint32_t B, uint32_t inactiveMask, const float *bias,
                                        uint32_t *counts, uint32_t countsStride, float presence, float frequency, cudaStream_t stream) {
    const dl::SampleControls ctl{bias, counts, countsStride, presence, frequency};
    return dl::launchSampleRows(logits, logitsStride, probsScratch, n, temperature, topp, rngState, tokenOut, B, inactiveMask, nullptr, nullptr, 1,
                                stream, &ctl);
}

// dl_sample_rows_controlled with per-row settings: rowParams (device f32 [B][4]) holds row b's {temperature, top-p, presence,
// frequency}; row b's bias (may be null) is bias + b * biasStride. A row with temperature 0 draws the arg-max.
DL_EXPORT int dl_sample_rows_per_row(const float *logits, uint32_t logitsStride, float *probsScratch, uint32_t n, const float *rowParams,
                                     unsigned long long *rngState, int *tokenOut, uint32_t B, uint32_t inactiveMask, const float *bias,
                                     uint32_t biasStride, uint32_t *counts, uint32_t countsStride, cudaStream_t stream) {
    dl::SampleControls ctl{bias, counts, countsStride, 0.f, 0.f, biasStride};
    return dl::launchSampleRows(logits, logitsStride, probsScratch, n, 0.f, 0.f, rngState, tokenOut, B, inactiveMask, nullptr, nullptr, 1, stream,
                                (bias || counts) ? &ctl : nullptr, rowParams);
}

// dl_sample_logits with the filters (kernels.h: SampleFilters) topK / minP.
DL_EXPORT int dl_sample_logits_filtered(const float *logits, float *probsScratch, uint32_t n, float temperature, float topp, uint32_t topK,
                                        float minP, unsigned long long *rngState, int *tokenOut, cudaStream_t stream) {
    const dl::SampleFilters f{topK, minP};
    return dl::launchSample(logits, probsScratch, n, temperature, topp, rngState, tokenOut, nullptr, nullptr, 0, nullptr, nullptr, 1, stream,
                            nullptr, &f);
}

// dl_sample_rows_per_row with per-row filters: rowFilters (device [B] {u32 topK, f32 minP}, may be null) holds row b's filters.
DL_EXPORT int dl_sample_rows_filtered(const float *logits, uint32_t logitsStride, float *probsScratch, uint32_t n, const float *rowParams,
                                      const void *rowFilters, unsigned long long *rngState, int *tokenOut, uint32_t B, uint32_t inactiveMask,
                                      const float *bias, uint32_t biasStride, uint32_t *counts, uint32_t countsStride, cudaStream_t stream) {
    dl::SampleControls ctl{bias, counts, countsStride, 0.f, 0.f, biasStride};
    return dl::launchSampleRows(logits, logitsStride, probsScratch, n, 0.f, 0.f, rngState, tokenOut, B, inactiveMask, nullptr, nullptr, 1, stream,
                                (bias || counts) ? &ctl : nullptr, rowParams, nullptr, (const dl::SampleFilters *)rowFilters);
}
