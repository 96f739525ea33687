// Decode attention of a slots step: B independent sequences, each in its own KV-cache slot, decoded in one batched forward.
//
// Slot layout (head-major bf16 cache of one layer, [nKvHeads][seqLen][headDim] split into equal slots): slot s is the contiguous
// [nKvHeads][L][headDim] block at element offset s * slotStride, slotStride = nKvHeads * L * headDim. Row b of the step is slot b;
// its token sits at position pos[b] and its K/V row pos[b] was written by ropeKvKernel (RopeKvArgs::slotStride) before this
// kernel runs. Row b attends to rows [0, pos[b]] of its own slot and nothing else.
//
// grid (nKvHeads, nSplits, B), block 128 (4 warps). CTA (kvh, split, b) stages 32-row tiles of K and V of its chunk in shared
// memory once and runs the kvMul q-heads of that KV head over them (one q-head per warp, round robin), so every K/V row is read
// once per (row, KV head). Inside a tile lane i scores position i; the online-softmax state (m, l, acc[HD]) of each q-head lives
// in shared memory between tiles. The number of effective splits follows from the row's own length, so a row's arithmetic does not
// depend on the other rows of the step. The last CTA of (b, kvh) to finish merges the splits in split order.
//
// Why a third decode-attention kernel: attnDecodeKernel runs one CTA per q-head and so reads each K/V row kvMul times (4 for
// Llama-3.1-8B); with 8 sequences at 2048 tokens that is about 64 MB of K/V per layer and step, more than the 50 MB L2.
// choiceAttnKernel packs the q-heads the same way but is built around one prefix shared by every row. Both keep serving their
// callers (single sequence and prefill; choices) unchanged.
#include "kernels.h"

namespace dl {
namespace {

constexpr int kTile = 32;

template <int HD>
struct SlotSmem {
    static constexpr int kRowPad = HD + 2;   // bf16 per staged row: the odd word stride keeps lane-per-row K reads conflict-free
    static size_t bytes(uint32_t R) {
        return (size_t)R * HD * 4 /* q */ + (size_t)R * HD * 4 /* acc */ + (size_t)R * 8 /* m, l */ + 2ull * kTile * kRowPad * 2;
    }
};

template <int HD>
__global__ void __launch_bounds__(128) slotAttnKernel(SlotAttnArgs a) {
    constexpr int DPL = HD / 32;
    constexpr int RP = SlotSmem<HD>::kRowPad;
    pdlLaunchDependents();
    pdlWait();
    const uint32_t kvh = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
    if (b < 32 && ((a.inactiveMask >> b) & 1u)) return;
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t R = a.nHeads / a.nKvHeads;                   // q-heads of this KV head
    float *sQ = reinterpret_cast<float *>(smem);                // [R][HD], pre-scaled by 1/sqrt(HD)
    float *sAcc = sQ + (size_t)R * HD;                          // [R][HD]
    float *sM = sAcc + (size_t)R * HD, *sL = sM + R;            // [R]
    __nv_bfloat16 *sK = reinterpret_cast<__nv_bfloat16 *>(sL + R);   // [kTile][RP]
    __nv_bfloat16 *sV = sK + kTile * RP;
    __shared__ bool sLast;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int p = a.pos[b];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.L) p = (int)a.L - 1;
    const uint32_t nPos = (uint32_t)p + 1;
    uint32_t eff = (nPos + 63) / 64;
    if (eff > a.nSplits) eff = a.nSplits;
    if (eff < 1) eff = 1;
    if (split >= eff) return;
    const uint32_t chunk = (nPos + eff - 1) / eff;
    const uint32_t begin = split * chunk, end = min(begin + chunk, nPos);

    const float scale = rsqrtf((float)HD);
    const float *qRow = a.qkv + (size_t)b * a.qkvStride + (size_t)kvh * R * HD;
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) { sQ[i] = qRow[i] * scale; sAcc[i] = 0.f; }
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { sM[r] = -INFINITY; sL[r] = 0.f; }

    const size_t headOff = (size_t)b * a.slotStride + (size_t)kvh * a.L * HD;
    const __nv_bfloat16 *kHead = a.kCache + headOff, *vHead = a.vCache + headOff;
    for (uint32_t t0 = begin; t0 < end; t0 += kTile) {
        const uint32_t len = min((uint32_t)kTile, end - t0);
        __syncthreads();   // the previous tile (and the initialisation above) is complete
        for (uint32_t i = threadIdx.x; i < kTile * (HD / 2); i += blockDim.x) {
            const uint32_t rr = i / (HD / 2), c = i % (HD / 2);
            __nv_bfloat162 kv = __floats2bfloat162_rn(0.f, 0.f), vv = kv;
            if (rr < len) {
                const size_t off = (size_t)(t0 + rr) * HD + 2 * c;
                kv = *reinterpret_cast<const __nv_bfloat162 *>(kHead + off);
                vv = *reinterpret_cast<const __nv_bfloat162 *>(vHead + off);
            }
            reinterpret_cast<__nv_bfloat162 *>(sK + rr * RP)[c] = kv;
            reinterpret_cast<__nv_bfloat162 *>(sV + rr * RP)[c] = vv;
        }
        __syncthreads();
        for (uint32_t r = warp; r < R; r += 4) {
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
    __syncthreads();

    float *outRow = a.out + (size_t)b * a.outStride + (size_t)kvh * R * HD;
    if (eff == 1) {
        for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) outRow[i] = sAcc[i] / sL[i / HD];
        return;
    }
    // partial of (b, kvh, split): [R][HD + 2] = (unnormalised acc, m, l)
    const size_t group = (size_t)b * a.nKvHeads + kvh;
    float *pOut = a.partial + (group * a.nSplits + split) * R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) pOut[(i / HD) * (HD + 2) + i % HD] = sAcc[i];
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { pOut[r * (HD + 2) + HD] = sM[r]; pOut[r * (HD + 2) + HD + 1] = sL[r]; }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counters[group], 1u);
        sLast = prev == eff - 1;
        if (sLast) a.counters[group] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const float *pIn = a.partial + group * a.nSplits * R * (HD + 2);
    const size_t splitStride = (size_t)R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
        const uint32_t r = i / HD, d = i % HD;
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
        outRow[i] = num / den;
    }
}

template <int HD>
int launchSlotAttnHd(const SlotAttnArgs &a, cudaStream_t stream, bool pdl) {
    const size_t smem = SlotSmem<HD>::bytes(a.nHeads / a.nKvHeads);
    static size_t configured = 0;
    if (smem > configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(slotAttnKernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    DL_CUDA_CHECK(launchPdl(slotAttnKernel<HD>, dim3(a.nKvHeads, a.nSplits, a.B), dim3(128), smem, stream, pdl, a));
    return 0;
}

}  // namespace

int launchSlotAttn(const SlotAttnArgs &a, cudaStream_t stream, bool pdl) {
    if (a.nKvHeads == 0 || a.nHeads % a.nKvHeads || a.nSplits < 1 || a.L < 1 || a.B < 1 || a.B > 32) return -1;
    if (a.headDim == 128) return launchSlotAttnHd<128>(a, stream, pdl);
    if (a.headDim == 64) return launchSlotAttnHd<64>(a, stream, pdl);
    return -1;
}

}  // namespace dl

// Stand-alone entry for tests and measurements: slotAttnKernel alone over q rows that are already normalised and rotated, with
// every row's K/V already in its slot. pos is a device [B] array.
DL_EXPORT int dl_slot_attn(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, uint32_t nHeads,
                           uint32_t nKvHeads, uint32_t headDim, uint32_t L, uint32_t nSplits, uint32_t B, uint32_t inactiveMask, float *partial,
                           unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::SlotAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.kCache = (const __nv_bfloat16 *)kCache; a.vCache = (const __nv_bfloat16 *)vCache;
    a.slotStride = (uint64_t)nKvHeads * L * headDim; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.L = L;
    a.nSplits = nSplits; a.B = B; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchSlotAttn(a, stream, false);
}
