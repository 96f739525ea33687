// Attention of a choices step: B sequences ("choices") continue one prompt, all at the same rotary position.
//
// Cache layout of a choices step (head-major bf16 cache, [nKvHeads][seqLen][headDim]): rows [0, P] hold the shared prompt;
// choice b owns rows [P + 1 + b * C, P + 1 + (b + 1) * C). Its j-th generated token sits at rotary position P + 1 + j and at
// cache row P + 1 + b * C + j (written by ropeKvKernel with rowStride = C before this kernel runs).
//
// grid (nKvHeads, nSplits), block 128 (4 warps). CTA (kvh, split) stages 32-row tiles of K and V of its prefix chunk in shared
// memory once and runs every query row of the KV head over them: R = B * kvMul rows, row r = b * kvMul + g is q-head
// kvh * kvMul + g of choice b. Inside a tile lane i scores position i; the online softmax state (m, l, acc[HD]) of every row
// lives in shared memory between tiles. The last effective split also attends each active choice to its own rows. Splits are
// merged by max / normaliser in split order by the last CTA of the KV head to finish, as attnDecodeKernel merges its splits.
#include "kernels.h"

namespace dl {
namespace {

constexpr int kTile = 32;

template <int HD>
struct ChoiceSmem {
    static constexpr int kRowPad = HD + 2;   // bf16 per staged row: the odd word stride keeps lane-per-row K reads conflict-free
    static size_t bytes(uint32_t R) {
        return (size_t)R * HD * 4 /* q */ + (size_t)R * HD * 4 /* acc */ + (size_t)R * 8 /* m, l */ + 2ull * kTile * kRowPad * 2;
    }
};

template <int HD>
__global__ void __launch_bounds__(128) choiceAttnKernel(ChoiceAttnArgs a) {
    constexpr int DPL = HD / 32;
    constexpr int RP = ChoiceSmem<HD>::kRowPad;
    pdlLaunchDependents();
    pdlWait();
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t kvMul = a.nHeads / a.nKvHeads, R = a.B * kvMul;
    float *sQ = reinterpret_cast<float *>(smem);                // [R][HD], pre-scaled by 1/sqrt(HD)
    float *sAcc = sQ + (size_t)R * HD;                          // [R][HD]
    float *sM = sAcc + (size_t)R * HD, *sL = sM + R;            // [R]
    __nv_bfloat16 *sK = reinterpret_cast<__nv_bfloat16 *>(sL + R);   // [kTile][RP]
    __nv_bfloat16 *sV = sK + kTile * RP;
    __shared__ bool sLast;

    const uint32_t kvh = blockIdx.x, split = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nPos = a.P + 1;
    uint32_t eff = (nPos + 63) / 64;
    if (eff > a.nSplits) eff = a.nSplits;
    if (eff < 1) eff = 1;
    if (split >= eff) return;
    const uint32_t chunk = (nPos + eff - 1) / eff;
    const uint32_t begin = split * chunk, end = min(begin + chunk, nPos);

    const float scale = rsqrtf((float)HD);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
        const uint32_t r = i / HD, d = i % HD, b = r / kvMul, h = kvh * kvMul + r % kvMul;
        sQ[i] = a.qkv[(size_t)b * a.qkvStride + (size_t)h * HD + d] * scale;
        sAcc[i] = 0.f;
    }
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { sM[r] = -INFINITY; sL[r] = 0.f; }

    const __nv_bfloat16 *kHead = a.kCache + (size_t)kvh * a.seqLen * HD;
    const __nv_bfloat16 *vHead = a.vCache + (size_t)kvh * a.seqLen * HD;
    // Cache rows [row0, row0 + n) for query rows [r0, r1): tiles of 32 rows, rows handed to the warps round robin.
    auto attend = [&](uint32_t row0, uint32_t n, uint32_t r0, uint32_t r1) {
        for (uint32_t t0 = 0; t0 < n; t0 += kTile) {
            const uint32_t len = min((uint32_t)kTile, n - t0);
            __syncthreads();   // the previous tile (and the initialisation above) is complete
            for (uint32_t i = threadIdx.x; i < kTile * (HD / 2); i += blockDim.x) {
                const uint32_t rr = i / (HD / 2), c = i % (HD / 2);
                __nv_bfloat162 kv = __floats2bfloat162_rn(0.f, 0.f), vv = kv;
                if (rr < len) {
                    const size_t off = (size_t)(row0 + t0 + rr) * HD + 2 * c;
                    kv = *reinterpret_cast<const __nv_bfloat162 *>(kHead + off);
                    vv = *reinterpret_cast<const __nv_bfloat162 *>(vHead + off);
                }
                reinterpret_cast<__nv_bfloat162 *>(sK + rr * RP)[c] = kv;
                reinterpret_cast<__nv_bfloat162 *>(sV + rr * RP)[c] = vv;
            }
            __syncthreads();
            for (uint32_t r = r0 + warp; r < r1; r += 4) {
                const float *q = sQ + (size_t)r * HD;
                const __nv_bfloat162 *kr = reinterpret_cast<const __nv_bfloat162 *>(sK + lane * RP);
                float s = 0.f;
#pragma unroll 8
                for (int c = 0; c < HD / 2; c++) {
                    const float2 k2 = __bfloat1622float2(kr[c]);
                    s += q[2 * c] * k2.x + q[2 * c + 1] * k2.y;
                }
                const bool valid = (uint32_t)lane < len;
                const float mOld = sM[r];
                const float mNew = fmaxf(mOld, warpMax(valid ? s : -INFINITY));
                const float corr = __expf(mOld - mNew);
                const float pr = valid ? __expf(s - mNew) : 0.f;
                const float lSum = warpSum(pr);
                float acc[DPL];
#pragma unroll
                for (int i = 0; i < DPL; i++) acc[i] = sAcc[(size_t)r * HD + lane * DPL + i] * corr;
                for (uint32_t u = 0; u < len; u++) {
                    const float pu = __shfl_sync(0xffffffffu, pr, u);
                    const __nv_bfloat16 *vr = sV + u * RP + lane * DPL;
#pragma unroll
                    for (int i = 0; i < DPL; i += 2) {
                        const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(vr + i));
                        acc[i] += pu * v2.x;
                        acc[i + 1] += pu * v2.y;
                    }
                }
#pragma unroll
                for (int i = 0; i < DPL; i++) sAcc[(size_t)r * HD + lane * DPL + i] = acc[i];
                __syncwarp();
                if (lane == 0) { sL[r] = sL[r] * corr + lSum; sM[r] = mNew; }
                __syncwarp();
            }
        }
    };
    attend(begin, end - begin, 0, R);
    if (split == eff - 1) {
        for (uint32_t b = 0; b < a.B; b++) {
            if ((a.inactiveMask >> b) & 1u) continue;
            attend(a.P + 1 + b * a.C, a.j + 1, b * kvMul, (b + 1) * kvMul);
        }
    }
    __syncthreads();

    if (eff == 1) {
        for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
            const uint32_t r = i / HD, d = i % HD, b = r / kvMul, h = kvh * kvMul + r % kvMul;
            a.out[(size_t)b * a.outStride + (size_t)h * HD + d] = sAcc[i] / sL[r];
        }
        return;
    }
    // partial of (kvh, split): [R][HD + 2] = (unnormalised acc, m, l)
    float *pOut = a.partial + ((size_t)kvh * a.nSplits + split) * R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) pOut[(i / HD) * (HD + 2) + i % HD] = sAcc[i];
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { pOut[r * (HD + 2) + HD] = sM[r]; pOut[r * (HD + 2) + HD + 1] = sL[r]; }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counters[kvh], 1u);
        sLast = prev == eff - 1;
        if (sLast) a.counters[kvh] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const float *pIn = a.partial + (size_t)kvh * a.nSplits * R * (HD + 2);
    const size_t splitStride = (size_t)R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
        const uint32_t r = i / HD, d = i % HD, b = r / kvMul, h = kvh * kvMul + r % kvMul;
        const float *pr = pIn + (size_t)r * (HD + 2);
        float gM = -INFINITY;
        for (uint32_t s = 0; s < eff; s++) gM = fmaxf(gM, __ldcg(pr + s * splitStride + HD));
        float num = 0.f, den = 0.f;
        for (uint32_t s = 0; s < eff; s++) {
            const float ms = __ldcg(pr + s * splitStride + HD);
            if (ms == -INFINITY) continue;
            const float w = __expf(ms - gM);
            num += w * __ldcg(pr + s * splitStride + d);
            den += w * __ldcg(pr + s * splitStride + HD + 1);
        }
        a.out[(size_t)b * a.outStride + (size_t)h * HD + d] = num / den;
    }
}

template <int HD>
int launchChoiceAttnHd(const ChoiceAttnArgs &a, cudaStream_t stream, bool pdl) {
    const size_t smem = ChoiceSmem<HD>::bytes(a.B * (a.nHeads / a.nKvHeads));
    static size_t configured = 0;
    if (smem > configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(choiceAttnKernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    DL_CUDA_CHECK(launchPdl(choiceAttnKernel<HD>, dim3(a.nKvHeads, a.nSplits), dim3(128), smem, stream, pdl, a));
    return 0;
}

}  // namespace

// Every active row's own rows [P + 1 + b * C, P + 1 + (b + 1) * C) lie inside the cache and j is inside them. Inactive rows
// (padding of the batch to a power of two) need no rows.
static bool choiceRowsFit(uint32_t B, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, uint32_t seqLen) {
    if (B < 1 || B > 32 || j >= C) return false;
    for (uint32_t b = 0; b < B; b++)
        if (!((inactiveMask >> b) & 1u) && (uint64_t)P + 1 + (uint64_t)(b + 1) * C > seqLen) return false;
    return true;
}

int launchChoiceAttn(const ChoiceAttnArgs &a, cudaStream_t stream, bool pdl) {
    if (a.nKvHeads == 0 || a.nHeads % a.nKvHeads || a.nSplits < 1) return -1;
    if (!choiceRowsFit(a.B, a.P, a.C, a.j, a.inactiveMask, a.seqLen)) return -1;
    if (a.headDim == 128) return launchChoiceAttnHd<128>(a, stream, pdl);
    if (a.headDim == 64) return launchChoiceAttnHd<64>(a, stream, pdl);
    return -1;
}

}  // namespace dl

// Stand-alone entry for tests: QK-norm + RoPE of B query rows at rotary position P + 1 + j, K/V append of the active rows at
// P + 1 + b * C + j (ropeKvKernel), then choiceAttnKernel. Every row of `pos` (device, [B]) must hold P + 1 + j.
DL_EXPORT int dl_choice_attn(float *qkv, uint32_t qkvStride, const int *pos, const float *rope, const float *qNorm, const float *kNorm, float eps,
                             void *kCache, void *vCache, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits,
                             uint32_t B, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, float *partial, unsigned int *counters,
                             float *out, uint32_t outStride, cudaStream_t stream) {
    dl::RopeKvArgs r{};
    r.qkv = qkv; r.qkvStride = qkvStride; r.pos = pos; r.rope = rope; r.qNorm = qNorm; r.kNorm = kNorm; r.eps = eps;
    r.nHeads = nHeads; r.nKvHeads = nKvHeads; r.headDim = headDim; r.seqLen = seqLen;
    r.kCache = (__nv_bfloat16 *)kCache; r.vCache = (__nv_bfloat16 *)vCache; r.rowStride = C; r.inactiveMask = inactiveMask;
    dl::ChoiceAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.kCache = r.kCache; a.vCache = r.vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.B = B; a.P = P; a.C = C; a.j = j; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    if (!dl::choiceRowsFit(B, P, C, j, inactiveMask, seqLen)) return -1;   // before anything is written
    const int rc = dl::launchRopeKv(r, (int)B, stream, false);
    if (rc != 0) return rc;
    return dl::launchChoiceAttn(a, stream, false);
}

// Stand-alone entry for measurements: choiceAttnKernel alone over q rows that are already normalised and rotated, with the
// choices' K/V rows already in the cache.
DL_EXPORT int dl_choice_attn_only(const float *qkv, uint32_t qkvStride, const void *kCache, const void *vCache, uint32_t nHeads, uint32_t nKvHeads,
                                  uint32_t headDim, uint32_t seqLen, uint32_t nSplits, uint32_t B, uint32_t P, uint32_t C, uint32_t j,
                                  uint32_t inactiveMask, float *partial, unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::ChoiceAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.kCache = (const __nv_bfloat16 *)kCache; a.vCache = (const __nv_bfloat16 *)vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.B = B; a.P = P; a.C = C; a.j = j; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchChoiceAttn(a, stream, false);
}
