// Small-batch (decode) kernels around the GEMVs: embedding gather, QK-norm + RoPE + KV-cache write, MoE router,
// greedy sampling. Decode attention is in attn_decode.cu.
//
// Reference ops replaced: OP_EMBEDDING (nn-cpu-ops.cpp:982-1008), OP_INV_RMS/OP_RMS_NORM per head
// (llm.cpp:322-346), OP_ROPE (nn-cpu-ops.cpp:843-885), OP_SHIFT (:1419-1441), host argmax (tokenizer.cpp:392-403).
// Differences by design: KV cache is bf16 and head-major [kvHead][pos][headDim] (reference: f32 [pos][kvDim]);
// both rotary conventions run as adjacent-pair rotation because NeoX-style heads are re-ordered at load.
#include <type_traits>

#include "kernels.h"

namespace dl {

// ---- embedding ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) embeddingKernel(const EmbTable table, const int *__restrict__ tokens,
                                                       float *__restrict__ x, uint32_t dim, uint32_t xStride, uint32_t vocab) {
    pdlLaunchDependents();
    pdlWait();
    const int t = blockIdx.x;
    int tok = tokens[t];
    if (tok < 0 || (uint32_t)tok >= vocab) tok = 0;
    const float4 *src = reinterpret_cast<const float4 *>(table.row((uint32_t)tok, dim));
    float4 *dst = reinterpret_cast<float4 *>(x + (size_t)t * xStride);
    for (uint32_t i = threadIdx.x; i < dim / 4; i += blockDim.x) dst[i] = src[i];
}

// ---- QK-norm + RoPE + KV write -------------------------------------------------------------------------
// grid (nHeads + 2*nKvHeads, nb), block headDim/2: thread j rotates pair (2j, 2j+1). Q8: the cache is q80 (a 32-value block is
// the pairs of 16 neighbouring threads). PAGED: the row goes to its physical row through the token's page table.
template <bool Q8, bool PAGED>
__global__ void __launch_bounds__(128) ropeKvKernel(typename std::conditional<PAGED, PagedRopeKvArgs, RopeKvArgs>::type a) {
    pdlLaunchDependents();
    pdlWait();
    __shared__ float red[4];
    const uint32_t head = blockIdx.x, t = blockIdx.y, j = threadIdx.x, hd = a.headDim;
    int p = a.pos[t];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.seqLen) p = a.seqLen - 1;
    float *row = a.qkv + (size_t)t * a.qkvStride + (size_t)head * hd;
    float2 v = reinterpret_cast<float2 *>(row)[j];
    const bool isQ = head < a.nHeads;
    const bool isK = !isQ && head < a.nHeads + a.nKvHeads;
    if (isQ || isK) {
        const float *nw = isQ ? a.qNorm : a.kNorm;
        if (nw) {
            float ss = warpSum(v.x * v.x + v.y * v.y);
            if ((j & 31) == 0) red[j >> 5] = ss;
            __syncthreads();
            float tot = 0.f;
            for (uint32_t w = 0; w < (hd / 2 + 31) / 32; w++) tot += red[w];
            const float inv = rsqrtf(tot / (float)hd + a.eps);
            const float2 w2 = reinterpret_cast<const float2 *>(nw)[j];
            v.x = w2.x * (v.x * inv);
            v.y = w2.y * (v.y * inv);
        }
        const float2 cs = reinterpret_cast<const float2 *>(a.rope)[(size_t)p * (hd / 2) + j];
        const float x0 = v.x * cs.x - v.y * cs.y;
        const float x1 = v.x * cs.y + v.y * cs.x;
        v.x = x0; v.y = x1;
    }
    uint32_t cacheRow;
    if constexpr (PAGED) cacheRow = pagedRow(a.pageTable + (size_t)t * a.pageTableStride, (uint32_t)p);
    else cacheRow = (uint32_t)p + t * a.rowStride;
    const bool inactive = t < 32 && ((a.inactiveMask >> t) & 1u);
    if (isQ) {
        reinterpret_cast<float2 *>(row)[j] = v;
    } else if (!inactive && cacheRow < a.seqLen) {   // (uniform over the block: every thread of the row's warps gets here)
        const uint32_t kvh = isK ? head - a.nHeads : head - a.nHeads - a.nKvHeads;
        const size_t e = t * a.slotStride + ((size_t)kvh * a.seqLen + cacheRow) * hd + 2 * j;
        if constexpr (Q8) {
            float f[2] = {v.x, v.y};
            roundStoreKv<2, true>(f, isK ? a.kCache : a.vCache, isK ? a.kScale : a.vScale, e, true);
        } else {
            __nv_bfloat16 *cache = reinterpret_cast<__nv_bfloat16 *>(isK ? a.kCache : a.vCache);
            *reinterpret_cast<__nv_bfloat162 *>(cache + e) = __floats2bfloat162_rn(v.x, v.y);
        }
    }
}

// ---- MoE router: rmsnorm + gate GEMV (f32) + softmax + top-k + renormalise ---------------------------------------
// Reference ops: MATMUL(block_moe_gate) + SOFTMAX + MOE_GATE (src/llm.cpp:432-449, nn-cpu-ops.cpp:900-916,1462-1492).
// grid (nExperts/8, nb), block 256: every warp produces one expert logit; the last CTA of a token selects the top-k
// (lowest index wins ties) and writes the routing weights softmax(top-k logits).
__global__ void __launch_bounds__(256) moeRouterKernel(RouterArgs a) {
    pdlLaunchDependents();
    pdlWait();
    extern __shared__ float sy[];      // [dim] normalised activations
    __shared__ float red[8];
    __shared__ bool sLast;
    const uint32_t t = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float4 *x4 = reinterpret_cast<const float4 *>(a.x + (size_t)t * a.dim);
    float ss = 0.f;
    for (uint32_t i = threadIdx.x; i < a.dim / 4; i += 256) {
        const float4 v = x4[i];
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warpSum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < 8; i++) tot += red[i];
    const float inv = rsqrtf(tot / (float)a.dim + a.eps);
    for (uint32_t i = threadIdx.x; i < a.dim / 4; i += 256) {
        const float4 v = x4[i];
        const float4 w = reinterpret_cast<const float4 *>(a.normW)[i];
        reinterpret_cast<float4 *>(sy)[i] = make_float4(w.x * (v.x * inv), w.y * (v.y * inv), w.z * (v.z * inv), w.w * (v.w * inv));
    }
    __syncthreads();
    const uint32_t e = blockIdx.x * 8 + warp;
    if (e < a.nExperts) {
        const float4 *g4 = reinterpret_cast<const float4 *>(a.gate + (size_t)e * a.dim);
        float d = 0.f;
        for (uint32_t i = lane; i < a.dim / 4; i += 32) {
            const float4 g = g4[i];
            const float4 y = reinterpret_cast<const float4 *>(sy)[i];
            d += g.x * y.x + g.y * y.y + g.z * y.z + g.w * y.w;
        }
        d = warpSum(d);
        if (lane == 0) a.logits[(size_t)t * a.nExperts + e] = d;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counter[t], 1u);
        sLast = prev == gridDim.x - 1;
        if (sLast) a.counter[t] = 0;
    }
    __syncthreads();
    if (!sLast || warp != 0) return;
    __threadfence();
    // single warp: iterative arg-max over <= 256 experts (8 per lane)
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const uint32_t idx = lane + 32 * j;
        v[j] = idx < a.nExperts ? __ldcg(a.logits + (size_t)t * a.nExperts + idx) : -INFINITY;
    }
    float selV[8];
    int selI[8];
    for (uint32_t kk = 0; kk < a.k; kk++) {
        float best = -INFINITY;
        int bi = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (v[j] > best) { best = v[j]; bi = lane + 32 * j; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        selV[kk] = best;
        selI[kk] = bi;
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (lane + 32 * j == bi) v[j] = -INFINITY;
    }
    if (lane == 0) {
        float sum = 0.f;
        for (uint32_t kk = 0; kk < a.k; kk++) sum += __expf(selV[kk] - selV[0]);
        for (uint32_t kk = 0; kk < a.k; kk++) {
            a.expertIdx[t * a.k + kk] = selI[kk];
            a.expertWeight[t * a.k + kk] = __expf(selV[kk] - selV[0]) / sum;
        }
    }
}

// ---- greedy sampling -----------------------------------------------------------------------------------------
// One CTA scans the logits row, writes the arg-max token for the next step and advances the position.
__global__ void __launch_bounds__(1024) argmaxAdvanceKernel(const float *__restrict__ logits, uint32_t vocab, int *tokenOut,
                                                            int *pos, int *history, uint32_t historyCap) {
    pdlLaunchDependents();
    pdlWait();
    __shared__ float sv[32];
    __shared__ int si[32];
    float best = -INFINITY;
    int bi = 0;
    for (uint32_t i = threadIdx.x; i < vocab; i += blockDim.x) {
        const float v = logits[i];
        if (v > best) { best = v; bi = (int)i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sv[threadIdx.x];
        bi = si[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (threadIdx.x == 0) {
            tokenOut[0] = bi;
            const int p = pos[0] + 1;
            pos[0] = p;
            if (history && (uint32_t)p < historyCap) history[p] = bi;
        }
    }
}

// One CTA per logits row: row b's arg-max over ids [0, vocab), lowest id among equal maxima, into out[b]. The verify step of a
// speculative round uses it after a STORE logits GEMV where the fused per-row arg-max does not fit shared memory.
__global__ void __launch_bounds__(1024) argmaxRowsKernel(const float *__restrict__ logits, uint32_t stride, uint32_t vocab, int *out) {
    pdlLaunchDependents();
    pdlWait();
    __shared__ float sv[32];
    __shared__ int si[32];
    const float *row = logits + (size_t)blockIdx.x * stride;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (uint32_t i = threadIdx.x; i < vocab; i += blockDim.x) {
        const float v = row[i];
        if (v > best || bi == 0x7fffffff) { best = v; bi = (int)i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sv[threadIdx.x];
        bi = si[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (threadIdx.x == 0) out[blockIdx.x] = bi;
    }
}

int launchArgmaxRows(const float *logits, uint32_t stride, uint32_t vocab, int nb, int *out, cudaStream_t stream, bool pdl) {
    if (nb < 1 || vocab < 1) return -1;
    DL_CUDA_CHECK(launchPdl(argmaxRowsKernel, dim3(nb), dim3(1024), 0, stream, pdl, logits, stride, vocab, out));
    return 0;
}

int launchEmbedding(const EmbTable &table, const int *tokens, float *x, uint32_t dim, uint32_t xStride, uint32_t vocab, int nb,
                    cudaStream_t stream) {
    embeddingKernel<<<nb, 256, 0, stream>>>(table, tokens, x, dim, xStride, vocab);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int launchRopeKv(const RopeKvArgs &a, int nb, cudaStream_t stream, bool pdl) {
    if (a.headDim != 64 && a.headDim != 128 && a.headDim != 256) return -1;
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    const dim3 grid(a.nHeads + 2 * a.nKvHeads, nb), block(a.headDim / 2);
    if (a.kScale) DL_CUDA_CHECK(launchPdl(ropeKvKernel<true, false>, grid, block, 0, stream, pdl, a));
    else DL_CUDA_CHECK(launchPdl(ropeKvKernel<false, false>, grid, block, 0, stream, pdl, a));
    return 0;
}

int launchRopeKvPaged(const PagedRopeKvArgs &a, int nb, cudaStream_t stream, bool pdl) {
    if (a.headDim != 64 && a.headDim != 128 && a.headDim != 256) return -1;
    if ((a.kScale == nullptr) != (a.vScale == nullptr) || !a.pageTable || a.slotStride || a.rowStride) return -1;
    const dim3 grid(a.nHeads + 2 * a.nKvHeads, nb), block(a.headDim / 2);
    if (a.kScale) DL_CUDA_CHECK(launchPdl(ropeKvKernel<true, true>, grid, block, 0, stream, pdl, a));
    else DL_CUDA_CHECK(launchPdl(ropeKvKernel<false, true>, grid, block, 0, stream, pdl, a));
    return 0;
}

int launchMoeRouter(const RouterArgs &a, int nb, cudaStream_t stream, bool pdl) {
    if (a.nExperts > 256 || a.k > 8 || a.dim % 4) return -1;
    DL_CUDA_CHECK(launchPdl(moeRouterKernel, dim3((a.nExperts + 7) / 8, nb), dim3(256), a.dim * sizeof(float), stream, pdl, a));
    return 0;
}

int launchArgmaxAdvance(const float *logits, uint32_t vocab, int *tokenOut, int *pos, int *history, uint32_t historyCap,
                        cudaStream_t stream, bool pdl) {
    DL_CUDA_CHECK(launchPdl(argmaxAdvanceKernel, dim3(1), dim3(1024), 0, stream, pdl, logits, vocab, tokenOut, pos, history, historyCap));
    return 0;
}

}  // namespace dl

// Stand-alone entry for the unit tests (tests/test_gpu_decode_attn.py): fills the argument struct and calls the launcher without
// programmatic dependent launch. Pointers are device pointers; caches are bf16 [nKvHeads][seqLen][headDim].
DL_EXPORT int dl_rope_kv(float *qkv, uint32_t qkvStride, const int *pos, const float *rope, const float *qNorm, const float *kNorm,
                         float eps, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, void *kCache, void *vCache,
                         int nb, cudaStream_t stream) {
    dl::RopeKvArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = kCache; a.vCache = vCache;
    return dl::launchRopeKv(a, nb, stream, false);
}

// dl_rope_kv into a q80 cache: int8 value planes kCache / vCache and f16 scale planes kScale / vScale [nKvHeads][seqLen][headDim / 32].
DL_EXPORT int dl_rope_kv_q80(float *qkv, uint32_t qkvStride, const int *pos, const float *rope, const float *qNorm, const float *kNorm,
                             float eps, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, void *kCache, void *vCache,
                             void *kScale, void *vScale, int nb, cudaStream_t stream) {
    dl::RopeKvArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = kCache; a.vCache = vCache; a.kScale = (__half *)kScale; a.vScale = (__half *)vScale;
    return dl::launchRopeKv(a, nb, stream, false);
}

// Greedy token of one logits row (tests/test_gpu_gemv.py): the lowest index among the maxima of logits[0, vocab) into tokenOut[0],
// pos[0] += 1 and history[pos] = token while pos < historyCap (history may be null).
DL_EXPORT int dl_argmax_advance(const float *logits, uint32_t vocab, int *tokenOut, int *pos, int *history, uint32_t historyCap,
                                cudaStream_t stream) {
    return dl::launchArgmaxAdvance(logits, vocab, tokenOut, pos, history, historyCap, stream, false);
}

// Router of T tokens (tests/test_gpu_moe.py): logits [T][nExperts], expertIdx / expertWeight [T][k]; counter [T] zeroed, self-resetting.
DL_EXPORT int dl_moe_router(const float *x, const float *normW, const float *gate, float eps, uint32_t dim, uint32_t nExperts, uint32_t k,
                            float *logits, unsigned int *counter, int *expertIdx, float *expertWeight, int T, cudaStream_t stream) {
    dl::RouterArgs a{};
    a.x = x; a.normW = normW; a.gate = gate; a.eps = eps; a.dim = dim; a.nExperts = nExperts; a.k = k;
    a.logits = logits; a.counter = counter; a.expertIdx = expertIdx; a.expertWeight = expertWeight;
    return dl::launchMoeRouter(a, T, stream, false);
}

// Per-row arg-max of nb logits rows (tests/test_gpu_speculative.py): row b = logits + b * stride, ids [0, vocab), into out[b].
DL_EXPORT int dl_argmax_rows(const float *logits, uint32_t stride, uint32_t vocab, int nb, int *out, cudaStream_t stream) {
    return dl::launchArgmaxRows(logits, stride, vocab, nb, out, stream, false);
}
