// Matrix-vector kernels for `.m` files whose matrices are *not* q40: f32 weights (the reference's F32_F32_F32 matmul
// with `--buffer-float-type f32`, src/nn/nn-cpu-ops.cpp:1138-1160, vulkan/matmul-forward-f32-f32-f32.comp) and f16
// weights (which the reference can store but not run). Activations stay f32 — no q80 round trip on this path.
//
// Same fusion contract as the q40 kernels (gemv_q40.cu): rmsnorm prologue, store / residual / SwiGLU epilogues,
// 1..8 tokens per launch, one persistent CTA per SM owning a contiguous pair-aligned row tile. The weight stream is
// 4-8x larger than q40, so the kernel is a pure streaming loop: every lane keeps kUnroll 16-byte loads in flight
// (64 KB per SM), activations are staged once per CTA in shared memory, row sums are reduced in a fixed order.
#include "gemv_common.cuh"

namespace dl {

namespace {

constexpr int kDenseThreads = 512;
constexpr int kDenseWarps = kDenseThreads / 32;
constexpr int kDenseUnroll = 8;

template <typename WT> struct Chunk;   // one 16-byte load of a weight row
template <> struct Chunk<float> {
    static constexpr int kElems = 4;
    __device__ static __forceinline__ void unpack(const uint4 &q, float (&w)[4]) {
        w[0] = __uint_as_float(q.x); w[1] = __uint_as_float(q.y); w[2] = __uint_as_float(q.z); w[3] = __uint_as_float(q.w);
    }
};
template <> struct Chunk<__half> {
    static constexpr int kElems = 8;
    __device__ static __forceinline__ void unpack(const uint4 &q, float (&w)[8]) {
        const uint32_t v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&v[i]));
            w[2 * i] = f.x; w[2 * i + 1] = f.y;
        }
    }
};

template <typename WT, int PRO, int EPI, int NB>
__global__ void __launch_bounds__(kDenseThreads, 1) gemvDenseKernel(GemvArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int E = Chunk<WT>::kElems;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    const uint32_t nPairs = a.d / 2;
    const uint32_t pairBegin = (uint32_t)(((uint64_t)blockIdx.x * nPairs) / gridDim.x);
    const uint32_t pairEnd = (uint32_t)(((uint64_t)(blockIdx.x + 1) * nPairs) / gridDim.x);
    const uint32_t rowBase = pairBegin * 2;
    const uint32_t tileRows = (pairEnd - pairBegin) * 2;

    float *xs = reinterpret_cast<float *>(smem);                 // [NB][n] (normalised) activations
    float *rowOut = xs + (size_t)NB * a.n;                       // [maxTileRows][NB]
    float *red = rowOut + (size_t)a.maxTileRows * NB;            // [16]

    pdlLaunchDependents();
    pdlWait();

    // ---- prologue: (rmsnorm) activations -> shared memory ----
    {
        const uint32_t nVec = a.n / 4;
#pragma unroll 1
        for (int t = 0; t < NB; t++) {
            const float4 *x4 = reinterpret_cast<const float4 *>(a.in + (size_t)t * a.inStride);
            float inv = 1.f;
            if (PRO == PRO_RMSNORM_) {
                float ss = 0.f;
                for (uint32_t i = tid; i < nVec; i += kDenseThreads) {
                    const float4 v = x4[i];
                    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
                }
                ss = blockSum512(ss, red);
                inv = rsqrtf(ss / (float)a.n + a.eps);
            }
            float4 *dst = reinterpret_cast<float4 *>(xs + (size_t)t * a.n);
            for (uint32_t i = tid; i < nVec; i += kDenseThreads) {
                float4 v = x4[i];
                if (PRO == PRO_RMSNORM_) v = rmsScale(v, reinterpret_cast<const float4 *>(a.normW)[i], inv);
                dst[i] = v;
            }
        }
    }
    __syncthreads();

    // ---- main loop: one warp per row, kDenseUnroll x 16 B in flight per lane ----
    const uint32_t nChunks = a.n / E;
    const WT *wBase = reinterpret_cast<const WT *>(a.qs);
    for (uint32_t r = warp; r < tileRows; r += kDenseWarps) {
        const uint4 *row = reinterpret_cast<const uint4 *>(wBase + (size_t)(rowBase + r) * a.n);
        float acc[NB];
#pragma unroll
        for (int t = 0; t < NB; t++) acc[t] = 0.f;
        for (uint32_t c0 = lane; c0 < nChunks; c0 += 32 * kDenseUnroll) {
            uint4 q[kDenseUnroll];
#pragma unroll
            for (int u = 0; u < kDenseUnroll; u++) {
                const uint32_t c = c0 + u * 32;
                q[u] = c < nChunks ? ldgStream16(row + c) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int u = 0; u < kDenseUnroll; u++) {
                const uint32_t c = c0 + u * 32;
                if (c < nChunks) {
                    float w[E];
                    Chunk<WT>::unpack(q[u], w);
#pragma unroll
                    for (int t = 0; t < NB; t++) {
                        const float4 *xv = reinterpret_cast<const float4 *>(xs + (size_t)t * a.n + (size_t)c * E);
#pragma unroll
                        for (int k = 0; k < E / 4; k++) {
                            const float4 x = xv[k];
                            acc[t] = fmaf(w[4 * k], x.x, acc[t]);
                            acc[t] = fmaf(w[4 * k + 1], x.y, acc[t]);
                            acc[t] = fmaf(w[4 * k + 2], x.z, acc[t]);
                            acc[t] = fmaf(w[4 * k + 3], x.w, acc[t]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int t = 0; t < NB; t++) {
            const float v = warpSum(acc[t]);
            if (lane == 0) rowOut[(size_t)r * NB + t] = v;
        }
    }
    __syncthreads();

    // ---- epilogue ----
    if (EPI == EPI_SWIGLU_) {
        const uint32_t tilePairs = tileRows / 2;
        for (uint32_t i = tid; i < tilePairs * NB; i += kDenseThreads) {
            const uint32_t p = i / NB, t = i - p * NB;
            const float g = rowOut[(size_t)(2 * p) * NB + t], up = rowOut[(size_t)(2 * p + 1) * NB + t];
            a.out[(size_t)t * a.outStride + pairBegin + p] = gateAct(g, a.act) * up;
        }
    } else {
        for (uint32_t i = tid; i < tileRows * NB; i += kDenseThreads) {
            const uint32_t r = i / NB, t = i - r * NB;
            float *o = a.out + (size_t)t * a.outStride + rowBase + r;
            const float v = rowOut[(size_t)r * NB + t];
            if (EPI == EPI_RESIDUAL_) *o += v;
            else *o = v;
        }
    }
}

// Expert-routed mode (mixture of experts, one token): the dense counterpart of the q40 TMA kernel's moeCtasPerSlot launches.
// The grid is kActive x moeCtasPerSlot; CTA b serves routing slot b / moeCtasPerSlot on the pair-aligned row tile
// b % moeCtasPerSlot of expert expertIdx[slot], so every slot uses the same tiling and the tiles line up for the combine.
//   PRO_RMSNORM_ + EPI_SWIGLU_ (W1|W3): rmsnorm(x) -> silu(gate) * up of slot s into out + s * outSlotStride.
//   PRO_PLAIN_ + EPI_MOE_DOWN_ (W2):    reads in + s * inSlotStride, leaves expertWeight[s] * product in moeScratch[s]; the
//                                       last CTA of a row tile (self-resetting moeCounters) adds sum_s moeScratch[s], summed in
//                                       slot order, to `out`: the result does not depend on which CTA finishes last.
// Under expert parallelism experts outside [moeFirstExpert, +moeNumLocal) stream nothing: their CTAs write zero products and
// still arrive at the combine counter. RPW rows per warp are streamed together with kMoeLoads / RPW 16-byte loads each, so
// short expert rows (a Qwen3-30B-A3B W2 row is 768 f16 values, 96 loads of a warp) still keep a lane's load slots full.
constexpr int kMoeLoads = 16;

template <typename WT, int PRO, int EPI, int RPW>
__global__ void __launch_bounds__(kDenseThreads, 1) gemvDenseMoeKernel(GemvArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int E = Chunk<WT>::kElems;
    constexpr int U = kMoeLoads / RPW;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    const uint32_t tileIdx = blockIdx.x % a.moeCtasPerSlot, slot = blockIdx.x / a.moeCtasPerSlot;
    const uint32_t nPairs = a.d / 2;
    const uint32_t pairBegin = (uint32_t)(((uint64_t)tileIdx * nPairs) / a.moeCtasPerSlot);
    const uint32_t pairEnd = (uint32_t)(((uint64_t)(tileIdx + 1) * nPairs) / a.moeCtasPerSlot);
    const uint32_t rowBase = pairBegin * 2;
    const uint32_t tileRows = (pairEnd - pairBegin) * 2;

    float *xs = reinterpret_cast<float *>(smem);                 // [n] (normalised) activations of this slot
    float *rowOut = xs + a.n;                                    // [maxTileRows]
    float *red = rowOut + a.maxTileRows;                         // [16]

    pdlLaunchDependents();
    pdlWait();   // the expert choice comes from the router, W2's input from the W1|W3 launch
    const uint32_t e = (uint32_t)a.expertIdx[slot] - a.moeFirstExpert;
    const bool active = e < a.moeNumLocal;

    if (active) {
        // ---- prologue: (rmsnorm) activations -> shared memory ----
        const uint32_t nVec = a.n / 4;
        const float4 *x4 = reinterpret_cast<const float4 *>(a.in + (size_t)slot * a.inSlotStride);
        float inv = 1.f;
        if (PRO == PRO_RMSNORM_) {
            float ss = 0.f;
            for (uint32_t i = tid; i < nVec; i += kDenseThreads) {
                const float4 v = x4[i];
                ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
            }
            ss = blockSum512(ss, red);
            inv = rsqrtf(ss / (float)a.n + a.eps);
        }
        float4 *dst = reinterpret_cast<float4 *>(xs);
        for (uint32_t i = tid; i < nVec; i += kDenseThreads) {
            float4 v = x4[i];
            if (PRO == PRO_RMSNORM_) v = rmsScale(v, reinterpret_cast<const float4 *>(a.normW)[i], inv);
            dst[i] = v;
        }
        __syncthreads();

        // ---- main loop: RPW adjacent rows per warp, U x 16 B in flight per lane and row ----
        const uint32_t nChunks = a.n / E;
        const WT *wBase = reinterpret_cast<const WT *>(a.qs) + (size_t)e * a.d * a.n;
        for (uint32_t r0 = warp * RPW; r0 < tileRows; r0 += kDenseWarps * RPW) {
            float acc[RPW];
#pragma unroll
            for (int j = 0; j < RPW; j++) acc[j] = 0.f;
            for (uint32_t c0 = lane; c0 < nChunks; c0 += 32 * U) {
                uint4 q[RPW][U];
#pragma unroll
                for (int j = 0; j < RPW; j++) {
                    const uint4 *row = reinterpret_cast<const uint4 *>(wBase + (size_t)(rowBase + r0 + j) * a.n);
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const uint32_t c = c0 + u * 32;
                        q[j][u] = (r0 + j < tileRows && c < nChunks) ? ldgStream16(row + c) : make_uint4(0, 0, 0, 0);
                    }
                }
#pragma unroll
                for (int j = 0; j < RPW; j++) {
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const uint32_t c = c0 + u * 32;
                        if (c < nChunks) {
                            float w[E];
                            Chunk<WT>::unpack(q[j][u], w);
                            const float4 *xv = reinterpret_cast<const float4 *>(xs + (size_t)c * E);
#pragma unroll
                            for (int k = 0; k < E / 4; k++) {
                                const float4 x = xv[k];
                                acc[j] = fmaf(w[4 * k], x.x, acc[j]);
                                acc[j] = fmaf(w[4 * k + 1], x.y, acc[j]);
                                acc[j] = fmaf(w[4 * k + 2], x.z, acc[j]);
                                acc[j] = fmaf(w[4 * k + 3], x.w, acc[j]);
                            }
                        }
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < RPW; j++) {
                const float v = warpSum(acc[j]);
                if (lane == 0 && r0 + j < tileRows) rowOut[r0 + j] = v;
            }
        }
    }
    __syncthreads();

    // ---- epilogue ----
    if (EPI == EPI_SWIGLU_) {
        float *outBase = a.out + (size_t)slot * a.outSlotStride;
        for (uint32_t p = tid; p < tileRows / 2; p += kDenseThreads)
            outBase[pairBegin + p] = active ? gateAct(rowOut[2 * p], a.act) * rowOut[2 * p + 1] : 0.f;
    } else {
        __shared__ bool sLastSlot;
        const float wgt = active ? a.expertWeight[slot] : 0.f;
        for (uint32_t i = tid; i < tileRows; i += kDenseThreads)
            a.moeScratch[(size_t)slot * a.d + rowBase + i] = active ? rowOut[i] * wgt : 0.f;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const unsigned int prev = atomicAdd(&a.moeCounters[tileIdx], 1u);
            sLastSlot = prev == a.kActive - 1;
            if (sLastSlot) a.moeCounters[tileIdx] = 0;
        }
        __syncthreads();
        if (!sLastSlot) return;
        __threadfence();
        for (uint32_t i = tid; i < tileRows; i += kDenseThreads) {
            float v = 0.f;
            for (uint32_t j = 0; j < a.kActive; j++) v += __ldcg(a.moeScratch + (size_t)j * a.d + rowBase + i);
            a.out[rowBase + i] += v;
        }
    }
}

template <auto Kernel>
int launchDense(const GemvArgs &a, int grid, size_t smemBytes, cudaStream_t stream, bool pdl) {
    DL_CUDA_CHECK(raiseSmemLimit<Kernel>(smemBytes));
    DL_CUDA_CHECK(launchPdl(Kernel, dim3(grid), dim3(kDenseThreads), smemBytes, stream, pdl, a));
    return 0;
}

template <typename WT>
int dispatchDenseMoe(int pro, int epi, int rpw, const GemvArgs &a, int grid, size_t smemBytes, cudaStream_t stream, bool pdl) {
#define DL_MOE_CASE(P, E, R) \
    if (pro == P && epi == E && rpw == R) return launchDense<gemvDenseMoeKernel<WT, P, E, R>>(a, grid, smemBytes, stream, pdl);
#define DL_MOE_RPW(P, E) DL_MOE_CASE(P, E, 1) DL_MOE_CASE(P, E, 2)
    DL_MOE_RPW(PRO_RMSNORM_, EPI_SWIGLU_)
    DL_MOE_RPW(PRO_PLAIN_, EPI_MOE_DOWN_)
    if constexpr (sizeof(WT) == 2) {   // four f32 rows of 4 loads each would spill: f32 stops at two rows per warp
        DL_MOE_CASE(PRO_RMSNORM_, EPI_SWIGLU_, 4)
        DL_MOE_CASE(PRO_PLAIN_, EPI_MOE_DOWN_, 4)
    }
#undef DL_MOE_RPW
#undef DL_MOE_CASE
    return -3;
}

template <typename WT>
int dispatchDense(int pro, int epi, int nb, const GemvArgs &a, int grid, size_t smemBytes, cudaStream_t stream, bool pdl) {
#define DL_DENSE_CASE(P, E, N) \
    if (pro == P && epi == E && nb == N) return launchDense<gemvDenseKernel<WT, P, E, N>>(a, grid, smemBytes, stream, pdl);
#define DL_DENSE_NB(P, E) DL_DENSE_CASE(P, E, 1) DL_DENSE_CASE(P, E, 2) DL_DENSE_CASE(P, E, 4) DL_DENSE_CASE(P, E, 8)
    DL_DENSE_NB(PRO_RMSNORM_, EPI_STORE_)
    DL_DENSE_NB(PRO_PLAIN_, EPI_RESIDUAL_)
    DL_DENSE_NB(PRO_RMSNORM_, EPI_SWIGLU_)
    DL_DENSE_NB(PRO_PLAIN_, EPI_STORE_)
#undef DL_DENSE_NB
#undef DL_DENSE_CASE
    return -3;
}

}  // namespace

size_t gemvDenseSmemBytes(uint32_t n, uint32_t maxTileRows, int nb) {
    return (size_t)nb * n * 4 + (size_t)maxTileRows * nb * 4 + 16 * 4 + 16;
}

// wtype: 1 = f32, 2 = f16. `a.qs` points at the row-major [d][n] matrix, `a.scales` is unused. Expert-routed launches
// (moeCtasPerSlot > 0, nb == 1) read `a.qs` as [moeNumLocal][d][n].
int gemvDense(int wtype, int pro, int epi, int nb, GemvArgs a, int numSms, cudaStream_t stream, bool pdl) {
    if (a.d % 2 || a.n % 8) return -1;
    a.act = gHiddenAct;
    if (a.ar.nRanks > 1) return -40;   // in-kernel all-reduce: q40 kernels only
    if (a.moeCtasPerSlot) {
        if (nb != 1 || !a.expertIdx || a.kActive == 0) return -41;
        const uint32_t nPairs = a.d / 2;
        const uint32_t tiles = a.moeCtasPerSlot < nPairs ? a.moeCtasPerSlot : nPairs;
        a.moeCtasPerSlot = tiles;
        a.maxTileRows = 2 * ((nPairs + tiles - 1) / tiles);
        const size_t smemBytes = gemvDenseSmemBytes(a.n, a.maxTileRows, 1);
        if (smemBytes > 227 * 1024) return -2;
        const uint32_t nChunks = a.n / (wtype == 1 ? 4 : 8);
        const int rpw = (wtype == 2 && nChunks <= 32 * (kMoeLoads / 4)) ? 4 : nChunks <= 32 * (kMoeLoads / 2) ? 2 : 1;
        const int grid = (int)(tiles * a.kActive);
        if (wtype == 1) return dispatchDenseMoe<float>(pro, epi, rpw, a, grid, smemBytes, stream, pdl);
        if (wtype == 2) return dispatchDenseMoe<__half>(pro, epi, rpw, a, grid, smemBytes, stream, pdl);
        return -4;
    }
    if (a.expertIdx) return -41;
    const uint32_t nPairs = a.d / 2;
    const int grid = (int)(nPairs < (uint32_t)numSms ? nPairs : (uint32_t)numSms);
    a.maxTileRows = 2 * ((nPairs + grid - 1) / grid);
    const size_t smemBytes = gemvDenseSmemBytes(a.n, a.maxTileRows, nb);
    if (smemBytes > 227 * 1024) return -2;
    if (wtype == 1) return dispatchDense<float>(pro, epi, nb, a, grid, smemBytes, stream, pdl);
    if (wtype == 2) return dispatchDense<__half>(pro, epi, nb, a, grid, smemBytes, stream, pdl);
    return -4;
}

}  // namespace dl

// Standalone entry points (tests / microbenchmarks). act: gate activation of EPI_SWIGLU (0 = SiLU, 1 = GELU).
DL_EXPORT int dl_gemv_dense(int wtype, int pro, int epi, int nb, const void *w, uint32_t d, uint32_t n, const float *in,
                            uint32_t inStride, const float *normW, float eps, float *out, uint32_t outStride, int numSms,
                            cudaStream_t stream, int pdl, uint32_t act) {
    const dl::HiddenActScope scope(act);
    dl::GemvArgs a{};
    a.qs = (const uint32_t *)w;
    a.d = d; a.n = n;
    a.in = in; a.normW = normW; a.eps = eps;
    a.out = out; a.inStride = inStride; a.outStride = outStride;
    return dl::gemvDense(wtype, pro, epi, nb, a, numSms, stream, pdl != 0);
}

// Shared memory a dense GEMV launch of nb tokens over a [d][n] matrix asks for (launches nothing); above 227 KB it is refused.
DL_EXPORT uint64_t dl_gemv_dense_smem_bytes(uint32_t d, uint32_t n, int nb, int numSms) {
    const uint32_t nPairs = d / 2;
    const uint32_t grid = nPairs < (uint32_t)numSms ? nPairs : (uint32_t)numSms;
    return dl::gemvDenseSmemBytes(n, 2 * ((nPairs + grid - 1) / grid), nb);
}
