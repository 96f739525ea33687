// Small-batch (decode) kernels around the GEMVs: embedding gather, QK-norm + RoPE + KV-cache write,
// split-KV attention with in-kernel merge, greedy sampling.
//
// Reference ops replaced: OP_EMBEDDING (nn-cpu-ops.cpp:982-1008), OP_INV_RMS/OP_RMS_NORM per head
// (llm.cpp:322-346), OP_ROPE (nn-cpu-ops.cpp:843-885), OP_SHIFT (:1419-1441), OP_MULTIHEAD_ATT (:753-788),
// host argmax (tokenizer.cpp:392-403).
// Differences by design: KV cache is bf16 and head-major [kvHead][pos][headDim] (reference: f32 [pos][kvDim]);
// both rotary conventions run as adjacent-pair rotation because NeoX-style heads are re-ordered at load;
// attention is flash-decoding (online softmax over KV splits, merged by the last CTA to finish).
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
// grid (nHeads + 2*nKvHeads, nb), block headDim/2: thread j rotates pair (2j, 2j+1)
__global__ void __launch_bounds__(128) ropeKvKernel(RopeKvArgs a) {
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
    const uint32_t cacheRow = (uint32_t)p + t * a.rowStride;
    const bool inactive = t < 32 && ((a.inactiveMask >> t) & 1u);
    if (isQ) {
        reinterpret_cast<float2 *>(row)[j] = v;
    } else if (!inactive && cacheRow < a.seqLen) {
        const uint32_t kvh = isK ? head - a.nHeads : head - a.nHeads - a.nKvHeads;
        __nv_bfloat16 *cache = isK ? a.kCache : a.vCache;
        __nv_bfloat162 *dst = reinterpret_cast<__nv_bfloat162 *>(cache + t * a.slotStride + ((size_t)kvh * a.seqLen + cacheRow) * hd);
        dst[j] = __floats2bfloat162_rn(v.x, v.y);
    }
}

// ---- decode attention ------------------------------------------------------------------------------------
// grid (nHeads, nSplits, nb), block 128 (4 warps). HD in {64, 128}.
template <int HD>
__global__ void __launch_bounds__(128) attnDecodeKernel(AttnArgs a) {
    constexpr int DPL = HD / 32;   // dims per lane
    pdlLaunchDependents();
    pdlWait();
    __shared__ float sAcc[4][HD];
    __shared__ float sM[4], sL[4];
    __shared__ bool sLast;
    const uint32_t h = blockIdx.x, split = blockIdx.y, t = blockIdx.z;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t kvh = h / (a.nHeads / a.nKvHeads);
    int p = a.pos[t];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.seqLen) p = a.seqLen - 1;
    const uint32_t nPos = (uint32_t)p + 1;
    const uint32_t chunk = (nPos + a.nSplits - 1) / a.nSplits;
    const uint32_t begin = split * chunk;
    const uint32_t end = min(begin + chunk, nPos);

    const float scale = rsqrtf((float)HD);
    float q[DPL];
    {
        const float *qrow = a.qkv + (size_t)t * a.qkvStride + (size_t)h * HD + lane * DPL;
#pragma unroll
        for (int i = 0; i < DPL; i++) q[i] = qrow[i] * scale;
    }
    const __nv_bfloat16 *kBase = a.kCache + (size_t)kvh * a.seqLen * HD + lane * DPL;
    const __nv_bfloat16 *vBase = a.vCache + (size_t)kvh * a.seqLen * HD + lane * DPL;

    float m = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) acc[i] = 0.f;

    constexpr int UN = 4;
    for (uint32_t s0 = begin + warp * UN; s0 < end; s0 += 4 * UN) {
        float kf[UN][DPL], vf[UN][DPL];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            const uint32_t s = s0 + u;
            if (s < end) {
                if constexpr (DPL == 4) {
                    const uint2 kr = *reinterpret_cast<const uint2 *>(kBase + (size_t)s * HD);
                    const uint2 vr = *reinterpret_cast<const uint2 *>(vBase + (size_t)s * HD);
                    const float2 k0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr.x));
                    const float2 k1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr.y));
                    const float2 v0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr.x));
                    const float2 v1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr.y));
                    kf[u][0] = k0.x; kf[u][1] = k0.y; kf[u][2] = k1.x; kf[u][3] = k1.y;
                    vf[u][0] = v0.x; vf[u][1] = v0.y; vf[u][2] = v1.x; vf[u][3] = v1.y;
                } else {
                    const uint32_t kr = *reinterpret_cast<const uint32_t *>(kBase + (size_t)s * HD);
                    const uint32_t vr = *reinterpret_cast<const uint32_t *>(vBase + (size_t)s * HD);
                    const float2 k0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr));
                    const float2 v0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr));
                    kf[u][0] = k0.x; kf[u][1] = k0.y;
                    vf[u][0] = v0.x; vf[u][1] = v0.y;
                }
            } else {
#pragma unroll
                for (int i = 0; i < DPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
            }
        }
        float sc[UN];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            float d = 0.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) d += q[i] * kf[u][i];
            sc[u] = warpSum(d);
        }
#pragma unroll
        for (int u = 0; u < UN; u++) {
            if (s0 + u < end) {
                const float mNew = fmaxf(m, sc[u]);
                const float corr = __expf(m - mNew);
                const float pr = __expf(sc[u] - mNew);
                l = l * corr + pr;
#pragma unroll
                for (int i = 0; i < DPL; i++) acc[i] = acc[i] * corr + pr * vf[u][i];
                m = mNew;
            }
        }
    }
    // combine the 4 warps
#pragma unroll
    for (int i = 0; i < DPL; i++) sAcc[warp][lane * DPL + i] = acc[i];
    if (lane == 0) { sM[warp] = m; sL[warp] = l; }
    __syncthreads();
    const float M = fmaxf(fmaxf(sM[0], sM[1]), fmaxf(sM[2], sM[3]));
    float *pOut = a.partial + (((size_t)t * a.nHeads + h) * a.nSplits + split) * (HD + 2);
    if (threadIdx.x < HD) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 4; w++) v += (sM[w] == -INFINITY) ? 0.f : sAcc[w][threadIdx.x] * __expf(sM[w] - M);
        pOut[threadIdx.x] = v;
    }
    if (threadIdx.x == 0) {
        float L = 0.f;
#pragma unroll
        for (int w = 0; w < 4; w++) L += (sM[w] == -INFINITY) ? 0.f : sL[w] * __expf(sM[w] - M);
        pOut[HD] = M;
        pOut[HD + 1] = L;
    }
    // last CTA of this (token, head) merges the splits
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counters[t * a.nHeads + h], 1u);
        sLast = (prev == a.nSplits - 1);
        if (sLast) a.counters[t * a.nHeads + h] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const float *pIn = a.partial + ((size_t)t * a.nHeads + h) * a.nSplits * (HD + 2);
    float gM = -INFINITY;
    for (uint32_t s = 0; s < a.nSplits; s++) gM = fmaxf(gM, __ldcg(pIn + (size_t)s * (HD + 2) + HD));
    if (threadIdx.x < HD) {
        float num = 0.f, den = 0.f;
        for (uint32_t s = 0; s < a.nSplits; s++) {
            const float ms = __ldcg(pIn + (size_t)s * (HD + 2) + HD);
            if (ms == -INFINITY) continue;
            const float w = __expf(ms - gM);
            num += w * __ldcg(pIn + (size_t)s * (HD + 2) + threadIdx.x);
            den += w * __ldcg(pIn + (size_t)s * (HD + 2) + HD + 1);
        }
        if (a.outBf16) a.outBf16[(size_t)t * a.outStride + (size_t)h * HD + threadIdx.x] = __float2bfloat16_rn(num / den);
        else a.out[(size_t)t * a.outStride + (size_t)h * HD + threadIdx.x] = num / den;
    }
}

// ---- fused single-token attention: QK-norm + RoPE + KV append + split-KV attention + merge --------------------
// grid (nHeads, nSplits), block 128. The number of *effective* splits is derived from the position on the device
// (>= 64 cached positions per split), so short contexts run as one CTA per head with no merge pass at all.
// The current token's K/V never round-trips through the cache: the split that covers position `pos` rotates k
// in registers; the first q-head of every KV group also appends k/v to the cache for later steps.
template <int HD>
__global__ void __launch_bounds__(128) attnFusedKernel(AttnFusedArgs a) {
    constexpr int DPL = HD / 32;
    static_assert(DPL == 2 || DPL == 4, "head dim must be 64 or 128");
    traceStamp(a.trace, 0);
    pdlLaunchDependents();
    pdlWait();
    traceStamp(a.trace, 1);
    __shared__ float sAcc[4][HD];
    __shared__ float sM[4], sL[4];
    __shared__ bool sLast;
    const uint32_t h = blockIdx.x, split = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t kvMul = a.nHeads / a.nKvHeads, kvh = h / kvMul;
    int p = a.pos[0];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.seqLen) p = a.seqLen - 1;
    const uint32_t nPos = (uint32_t)p + 1;
    uint32_t eff = (nPos + 63) / 64;
    if (eff > a.nSplits) eff = a.nSplits;
    if (eff < 1) eff = 1;
    if (split >= eff) return;
    const uint32_t chunk = (nPos + eff - 1) / eff;
    const uint32_t begin = split * chunk;
    const uint32_t end = min(begin + chunk, nPos);
    const bool ownsNew = end == nPos;                    // this split covers the token being generated
    const uint32_t cachedEnd = ownsNew ? end - 1 : end;  // positions read from the cache: [begin, cachedEnd)

    const uint32_t qDim = a.nHeads * HD, kvDim = a.nKvHeads * HD;
    const float2 *ropeRow = reinterpret_cast<const float2 *>(a.rope) + (size_t)p * (HD / 2) + lane * (DPL / 2);
    auto normRope = [&](float *v, const float *nw) {
        if (nw) {
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) ss += v[i] * v[i];
            ss = warpSum(ss);
            const float inv = rsqrtf(ss / (float)HD + a.eps);
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

    float q[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) q[i] = a.qkv[(size_t)h * HD + lane * DPL + i];
    normRope(q, a.qNorm);
    const float scale = rsqrtf((float)HD);
#pragma unroll
    for (int i = 0; i < DPL; i++) q[i] *= scale;

    float m = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) acc[i] = 0.f;

    __nv_bfloat16 *kHead = a.kCache + (size_t)kvh * a.seqLen * HD;
    __nv_bfloat16 *vHead = a.vCache + (size_t)kvh * a.seqLen * HD;
    if (ownsNew && warp == 0) {
        float kn[DPL], vn[DPL];
#pragma unroll
        for (int i = 0; i < DPL; i++) {
            kn[i] = a.qkv[qDim + (size_t)kvh * HD + lane * DPL + i];
            vn[i] = a.qkv[qDim + kvDim + (size_t)kvh * HD + lane * DPL + i];
        }
        normRope(kn, a.kNorm);
        // the cache holds bf16: use the rounded values here too so this step matches what later steps will read
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
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < DPL; i++) d += q[i] * kn[i];
        d = warpSum(d);
        m = d; l = 1.f;
#pragma unroll
        for (int i = 0; i < DPL; i++) acc[i] = vn[i];
    }

    const __nv_bfloat16 *kBase = kHead + lane * DPL;
    const __nv_bfloat16 *vBase = vHead + lane * DPL;
    constexpr int UN = 4;
    for (uint32_t s0 = begin + warp * UN; s0 < cachedEnd; s0 += 4 * UN) {
        float kf[UN][DPL], vf[UN][DPL];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            const uint32_t s = s0 + u;
            if (s < cachedEnd) {
                if constexpr (DPL == 4) {
                    const uint2 kr = *reinterpret_cast<const uint2 *>(kBase + (size_t)s * HD);
                    const uint2 vr = *reinterpret_cast<const uint2 *>(vBase + (size_t)s * HD);
                    const float2 k0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr.x));
                    const float2 k1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr.y));
                    const float2 v0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr.x));
                    const float2 v1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr.y));
                    kf[u][0] = k0.x; kf[u][1] = k0.y; kf[u][2] = k1.x; kf[u][3] = k1.y;
                    vf[u][0] = v0.x; vf[u][1] = v0.y; vf[u][2] = v1.x; vf[u][3] = v1.y;
                } else {
                    const uint32_t kr = *reinterpret_cast<const uint32_t *>(kBase + (size_t)s * HD);
                    const uint32_t vr = *reinterpret_cast<const uint32_t *>(vBase + (size_t)s * HD);
                    const float2 k0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&kr));
                    const float2 v0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&vr));
                    kf[u][0] = k0.x; kf[u][1] = k0.y;
                    vf[u][0] = v0.x; vf[u][1] = v0.y;
                }
            } else {
#pragma unroll
                for (int i = 0; i < DPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
            }
        }
        float sc[UN];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            float d = 0.f;
#pragma unroll
            for (int i = 0; i < DPL; i++) d += q[i] * kf[u][i];
            sc[u] = warpSum(d);
        }
#pragma unroll
        for (int u = 0; u < UN; u++) {
            if (s0 + u < cachedEnd) {
                const float mNew = fmaxf(m, sc[u]);
                const float corr = __expf(m - mNew);
                const float pr = __expf(sc[u] - mNew);
                l = l * corr + pr;
#pragma unroll
                for (int i = 0; i < DPL; i++) acc[i] = acc[i] * corr + pr * vf[u][i];
                m = mNew;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < DPL; i++) sAcc[warp][lane * DPL + i] = acc[i];
    if (lane == 0) { sM[warp] = m; sL[warp] = l; }
    __syncthreads();
    const float M = fmaxf(fmaxf(sM[0], sM[1]), fmaxf(sM[2], sM[3]));
    float num = 0.f, L = 0.f;
    if (threadIdx.x < HD) {
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const float wgt = (sM[w] == -INFINITY) ? 0.f : __expf(sM[w] - M);
            num += sAcc[w][threadIdx.x] * wgt;
            L += sL[w] * wgt;
        }
    }
    float *outRow = a.out + (size_t)h * HD;
    if (eff == 1) {
        if (threadIdx.x < HD) outRow[threadIdx.x] = num / L;
        traceStamp(a.trace, 3);
        return;
    }
    float *pOut = a.partial + ((size_t)h * a.nSplits + split) * (HD + 2);
    if (threadIdx.x < HD) pOut[threadIdx.x] = num;
    if (threadIdx.x == 0) { pOut[HD] = M; pOut[HD + 1] = L; }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counters[h], 1u);
        sLast = (prev == eff - 1);
        if (sLast) a.counters[h] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const float *pIn = a.partial + (size_t)h * a.nSplits * (HD + 2);
    float gM = -INFINITY;
    for (uint32_t s = 0; s < eff; s++) gM = fmaxf(gM, __ldcg(pIn + (size_t)s * (HD + 2) + HD));
    if (threadIdx.x < HD) {
        float n2 = 0.f, den = 0.f;
        for (uint32_t s = 0; s < eff; s++) {
            const float ms = __ldcg(pIn + (size_t)s * (HD + 2) + HD);
            const float w = __expf(ms - gM);
            n2 += w * __ldcg(pIn + (size_t)s * (HD + 2) + threadIdx.x);
            den += w * __ldcg(pIn + (size_t)s * (HD + 2) + HD + 1);
        }
        outRow[threadIdx.x] = n2 / den;
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

int launchEmbedding(const EmbTable &table, const int *tokens, float *x, uint32_t dim, uint32_t xStride, uint32_t vocab, int nb,
                    cudaStream_t stream) {
    embeddingKernel<<<nb, 256, 0, stream>>>(table, tokens, x, dim, xStride, vocab);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

template <typename K, typename A>
static int launchPdl(K kernel, dim3 grid, dim3 block, cudaStream_t stream, bool pdl, const A &args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, args));
    return 0;
}

int launchRopeKv(const RopeKvArgs &a, int nb, cudaStream_t stream, bool pdl) {
    if (a.headDim != 64 && a.headDim != 128 && a.headDim != 256) return -1;
    return launchPdl(ropeKvKernel, dim3(a.nHeads + 2 * a.nKvHeads, nb), dim3(a.headDim / 2), stream, pdl, a);
}

int launchAttnDecode(const AttnArgs &a, int nb, cudaStream_t stream, bool pdl) {
    const dim3 grid(a.nHeads, a.nSplits, nb);
    if (a.headDim == 128) return launchPdl(attnDecodeKernel<128>, grid, dim3(128), stream, pdl, a);
    if (a.headDim == 64) return launchPdl(attnDecodeKernel<64>, grid, dim3(128), stream, pdl, a);
    return -1;
}

int launchMoeRouter(const RouterArgs &a, int nb, cudaStream_t stream, bool pdl) {
    if (a.nExperts > 256 || a.k > 8 || a.dim % 4) return -1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((a.nExperts + 7) / 8, nb);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = a.dim * sizeof(float);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, moeRouterKernel, a));
    return 0;
}

int launchAttnFused(const AttnFusedArgs &a, cudaStream_t stream, bool pdl) {
    const dim3 grid(a.nHeads, a.nSplits);
    if (a.headDim == 128) return launchPdl(attnFusedKernel<128>, grid, dim3(128), stream, pdl, a);
    if (a.headDim == 64) return launchPdl(attnFusedKernel<64>, grid, dim3(128), stream, pdl, a);
    return -1;
}

int launchArgmaxAdvance(const float *logits, uint32_t vocab, int *tokenOut, int *pos, int *history, uint32_t historyCap,
                        cudaStream_t stream, bool pdl) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(1);
    cfg.blockDim = dim3(1024);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, argmaxAdvanceKernel, logits, vocab, tokenOut, pos, history, historyCap));
    return 0;
}

}  // namespace dl

// Stand-alone entry points for the unit tests (tests/test_gpu_decode_attn.py): each fills the argument struct and calls the
// launcher without programmatic dependent launch. Pointers are device pointers; caches are bf16 [nKvHeads][seqLen][headDim].
DL_EXPORT int dl_rope_kv(float *qkv, uint32_t qkvStride, const int *pos, const float *rope, const float *qNorm, const float *kNorm,
                         float eps, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, void *kCache, void *vCache,
                         int nb, cudaStream_t stream) {
    dl::RopeKvArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen;
    a.kCache = (__nv_bfloat16 *)kCache; a.vCache = (__nv_bfloat16 *)vCache;
    return dl::launchRopeKv(a, nb, stream, false);
}

DL_EXPORT int dl_attn_decode(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, uint32_t nHeads,
                             uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits, float *partial, unsigned int *counters,
                             float *out, uint32_t outStride, void *outBf16, int nb, cudaStream_t stream) {
    dl::AttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos;
    a.kCache = (const __nv_bfloat16 *)kCache; a.vCache = (const __nv_bfloat16 *)vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride; a.outBf16 = (__nv_bfloat16 *)outBf16;
    return dl::launchAttnDecode(a, nb, stream, false);
}

// Router of T tokens (tests/test_gpu_moe.py): logits [T][nExperts], expertIdx / expertWeight [T][k]; counter [T] zeroed, self-resetting.
DL_EXPORT int dl_moe_router(const float *x, const float *normW, const float *gate, float eps, uint32_t dim, uint32_t nExperts, uint32_t k,
                            float *logits, unsigned int *counter, int *expertIdx, float *expertWeight, int T, cudaStream_t stream) {
    dl::RouterArgs a{};
    a.x = x; a.normW = normW; a.gate = gate; a.eps = eps; a.dim = dim; a.nExperts = nExperts; a.k = k;
    a.logits = logits; a.counter = counter; a.expertIdx = expertIdx; a.expertWeight = expertWeight;
    return dl::launchMoeRouter(a, T, stream, false);
}

DL_EXPORT int dl_attn_fused(const float *qkv, const int *pos, const float *rope, const float *qNorm, const float *kNorm, float eps,
                            void *kCache, void *vCache, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen,
                            uint32_t nSplits, float *partial, unsigned int *counters, float *out, cudaStream_t stream) {
    dl::AttnFusedArgs a{};
    a.qkv = qkv; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.kCache = (__nv_bfloat16 *)kCache; a.vCache = (__nv_bfloat16 *)vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out;
    return dl::launchAttnFused(a, stream, false);
}
