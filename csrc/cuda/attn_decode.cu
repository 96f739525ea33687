// Decode attention: a few query tokens against the head-major KV cache ([nKvHeads][seqLen][headDim]), flash-decoding style
// (online softmax over KV splits, merged in split order by the last CTA to finish). Reference op: OP_MULTIHEAD_ATT
// (nn-cpu-ops.cpp:753-788). Every kernel is instantiated for both cache storages (template parameter Q8, see kernels.h): bf16 rows,
// or q80 rows dequantised on load; the q.k and p.v math is f32 either way.
//
// Four kernels, built from the shared pieces of the anonymous namespace below:
// * attnDecodeKernel: one CTA per (q-head, split, token), K/V rows streamed through registers. The GEMV-path batch and the
//   prefill fallback.
// * attnFusedKernel: one token, with QK-norm + RoPE + K/V append fused in. The multi-kernel single-token path.
// * choiceAttnKernel: the B choices of one prompt. One CTA per (KV head, split) over 32-row K/V tiles in shared memory.
// * slotAttnKernel: B independent sequences in KV-cache slots. One CTA per (KV head, split, row) over the same tiles.
//
// Every split of a group of R query rows writes its partial [R][HD + 2] = (unnormalised acc, m, l) and counts itself in the group's
// counter; the last one to arrive merges (finishSplit, written out in attnFusedKernel).
//
// Why the tile kernels pack the q-heads of a KV head onto one CTA: attnDecodeKernel runs one CTA per q-head and so reads each K/V
// row kvMul times (4 for Llama-3.1-8B); with 8 sequences at 2048 tokens that is about 64 MB of K/V per layer and step, more than
// the 50 MB L2. choiceAttnKernel reads each prompt row once per step for all the choices; slotAttnKernel reads each row once per
// (row, KV head).
//
// Cache layout of a choices step: rows [0, P] hold the shared prompt; choice b owns rows [P + 1 + b * C, P + 1 + (b + 1) * C). Its
// j-th generated token sits at rotary position P + 1 + j and at cache row P + 1 + b * C + j (written by ropeKvKernel with
// rowStride = C before choiceAttnKernel runs).
//
// Slot layout of a slots step: the layer's cache is split into equal slots; slot s is the contiguous [nKvHeads][L][headDim] block at
// element offset s * slotStride, slotStride = nKvHeads * L * headDim. Row b of the step is slot b; its token sits at position pos[b]
// and its K/V row pos[b] was written by ropeKvKernel (RopeKvArgs::slotStride) before slotAttnKernel runs. Row b attends to rows
// [0, pos[b]] of its own slot and nothing else.
//
// Paged slots (SlotAttnArgs::pageTable): every layer plane is one pool of 64-row pages, and slot b's logical row r lives at physical
// row table[b][r / 64] * 64 + r % 64 of the plane. slotAttnKernel stages the same 32-row tiles as for a contiguous slot, each row from
// its own page, so a step computes bit for bit what it computes in the contiguous layout.
#include <type_traits>

#include "kernels.h"

namespace dl {
namespace {

// The value plane of a cache (bf16, or int8 for Q8) advanced by `elems` elements.
template <bool Q8, typename P>
__device__ __forceinline__ P *kvPlane(P *plane, size_t elems) {
    using B = typename std::conditional<std::is_const<P>::value, const uint8_t, uint8_t>::type;
    return reinterpret_cast<B *>(plane) + elems * (Q8 ? 1 : 2);
}

// Split `split` when the number of splits follows from the length: ceil(nPos / 64) of them, at most nSplits, so short contexts run
// as one CTA per group with no merge pass. A row's splits depend on its own length only.
struct SplitRange {
    uint32_t eff, begin, end;
};
__device__ __forceinline__ SplitRange effectiveSplit(uint32_t nPos, uint32_t nSplits, uint32_t split) {
    uint32_t eff = (nPos + 63) / 64;
    if (eff > nSplits) eff = nSplits;
    if (eff < 1) eff = 1;
    const uint32_t chunk = (nPos + eff - 1) / eff;
    const uint32_t begin = split * chunk;
    return {eff, begin, min(begin + chunk, nPos)};
}

// Online softmax of one query head over cache rows [begin, end), K/V streamed through registers: each warp takes UN = 4 rows at a
// time, the 4 warps round robin, and lane i holds dims [i * DPL, (i + 1) * DPL). kHead / vHead (and kSc / vSc, Q8) point at the
// KV head's row 0.
template <int HD, bool Q8>
__device__ __forceinline__ void scanRows(const void *kHead, const void *vHead, const __half *kSc, const __half *vSc, const float (&q)[HD / 32],
                                         uint32_t begin, uint32_t end, float &m, float &l, float (&acc)[HD / 32]) {
    constexpr int DPL = HD / 32, UN = 4;
    const int warp = threadIdx.x >> 5;
    const uint32_t d0 = (threadIdx.x & 31) * DPL;
    for (uint32_t s0 = begin + warp * UN; s0 < end; s0 += 4 * UN) {
        float kf[UN][DPL], vf[UN][DPL];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            const uint32_t s = s0 + u;
            if (s < end) {
                loadKv<DPL, Q8>(kHead, kSc, (size_t)s * HD + d0, kf[u]);
                loadKv<DPL, Q8>(vHead, vSc, (size_t)s * HD + d0, vf[u]);
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
}

// Folds the online-softmax states of the 4 warps into the CTA's and returns its max M. Thread d < HD gets the unnormalised output
// element d in num and the normaliser in L. A warp that saw no row (m = -INFINITY) weighs 0. kFma picks how the weighted sums
// round: one fused multiply-add per warp (attnFusedKernel) or a rounded product and an add (attnDecodeKernel); each kernel keeps
// its own rounding so that its results do not move by a bit.
template <int HD, bool kFma>
__device__ __forceinline__ float combineWarps(float m, float l, const float (&acc)[HD / 32], float &num, float &L) {
    constexpr int DPL = HD / 32;
    __shared__ float sAcc[4][HD];
    __shared__ float sM[4], sL[4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < DPL; i++) sAcc[warp][lane * DPL + i] = acc[i];
    if (lane == 0) { sM[warp] = m; sL[warp] = l; }
    __syncthreads();
    const float M = fmaxf(fmaxf(sM[0], sM[1]), fmaxf(sM[2], sM[3]));
    num = 0.f;
    L = 0.f;
    if (threadIdx.x < HD) {
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const float wgt = (sM[w] == -INFINITY) ? 0.f : __expf(sM[w] - M);
            if constexpr (kFma) {
                num += sAcc[w][threadIdx.x] * wgt;
                L += sL[w] * wgt;
            } else {
                num += __fmul_rn(sAcc[w][threadIdx.x], wgt);
                L += __fmul_rn(sL[w], wgt);
            }
        }
    }
    return M;
}

// Ends split `split` of group `group`, R query rows split eff ways. The split's partial [R][HD + 2] goes to
// partial + (group * nSplits + split) * R * (HD + 2): acc(i) is its unnormalised element i = r * HD + d and ml(r) row r's (m, l).
// The last CTA of the group to arrive takes counters[group], resets it for the next launch and merges the splits in split order;
// store(i, v) writes merged element i. A split that saw no row (m = -INFINITY, acc = l = 0) is skipped by its weight:
// __expf(-INFINITY - gM) = 0 adds an exact +0 to both sums. A branch on m would make each split's loads wait for its m.
template <int HD, typename Acc, typename Ml, typename Store>
__device__ __forceinline__ void finishSplit(float *partial, unsigned int *counters, size_t group, uint32_t nSplits, uint32_t R,
                                            uint32_t split, uint32_t eff, Acc acc, Ml ml, Store store) {
    __shared__ bool sLast;
    partial += group * nSplits * R * (HD + 2);
    float *pOut = partial + (size_t)split * R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) pOut[(i / HD) * (HD + 2) + i % HD] = acc(i);
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) {
        const float2 s = ml(r);
        pOut[r * (HD + 2) + HD] = s.x;
        pOut[r * (HD + 2) + HD + 1] = s.y;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&counters[group], 1u);
        sLast = prev == eff - 1;
        if (sLast) counters[group] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const size_t splitStride = (size_t)R * (HD + 2);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
        const float *pr = partial + (size_t)(i / HD) * (HD + 2);
        const uint32_t d = i % HD;
        float gM = -INFINITY;
        for (uint32_t s = 0; s < eff; s++) gM = fmaxf(gM, __ldcg(pr + s * splitStride + HD));
        float num = 0.f, den = 0.f;
        for (uint32_t s = 0; s < eff; s++) {
            const float ms = __ldcg(pr + s * splitStride + HD);
            const float w = __expf(ms - gM);
            num += w * __ldcg(pr + s * splitStride + d);
            den += w * __ldcg(pr + s * splitStride + HD + 1);
        }
        store(i, num / den);
    }
}

constexpr int kTile = 32;   // K/V rows per shared-memory tile

// Dynamic shared memory of a tile kernel with R query rows: q [R][HD] (pre-scaled by 1/sqrt(HD)), the online-softmax state acc
// [R][HD], m [R] and l [R], then one K and one V tile of kTile rows. A bf16 cache is staged as bf16; a q80 one is widened to f32 on
// the way in (q * d needs more mantissa than bf16 has).
template <int HD, bool Q8>
struct TileSmem {
    using T = typename std::conditional<Q8, float, __nv_bfloat16>::type;
    // elements per staged row: the odd word stride keeps lane-per-row K reads conflict-free
    static constexpr int kRowPad = Q8 ? HD + 1 : HD + 2;
    float *q, *acc, *m, *l;
    T *k, *v;
    __device__ TileSmem(unsigned char *smem, uint32_t R)
        : q(reinterpret_cast<float *>(smem)), acc(q + (size_t)R * HD), m(acc + (size_t)R * HD), l(m + R),
          k(reinterpret_cast<T *>(l + R)), v(k + kTile * kRowPad) {}
    static size_t bytes(uint32_t R) {
        return (size_t)R * HD * 4 /* q */ + (size_t)R * HD * 4 /* acc */ + (size_t)R * 8 /* m, l */ + 2ull * kTile * kRowPad * sizeof(T);
    }
};

// The cache row of logical row r where rows are where they are (every layout but paged slots).
struct SameRow {
    __device__ __forceinline__ SameRow tile(uint32_t, uint32_t) const { return *this; }
    __device__ __forceinline__ uint32_t operator()(uint32_t r) const { return r; }
};
// The physical rows of a tile of a paged slot: its (at most two) pages, looked up once for the whole tile.
struct TilePages {
    uint32_t page0, row0, row1;   // the first row's logical page; physical row 0 of that page and of the next
    __device__ __forceinline__ uint32_t operator()(uint32_t r) const { return (r / kPageRows == page0 ? row0 : row1) + r % kPageRows; }
};
// The pages of a paged slot.
struct PagedRows {
    const int32_t *table;
    // rows [first, first + n)
    __device__ __forceinline__ TilePages tile(uint32_t first, uint32_t n) const {
        const uint32_t p0 = first / kPageRows, row0 = (uint32_t)__ldg(table + p0) * kPageRows;
        return {p0, row0, (first + n - 1) / kPageRows != p0 ? (uint32_t)__ldg(table + p0 + 1) * kPageRows : row0};
    }
};

// Query rows [r0, r1) attend to cache rows [row0, row0 + n) of one KV head (kHead / vHead, and kSc / vSc for Q8, point at its row 0).
// The rows are staged kTile at a time; inside a tile lane i scores row i, and the query rows go to the warps round robin. The rows
// of a tile are read from cache rows rowOf.tile(...)(row): a paged slot stages the same tiles from wherever its pages are (a tile
// may span two pages: splits need not start on a page edge), so the arithmetic does not depend on the layout.
template <int HD, bool Q8, typename RowOf = SameRow>
__device__ __forceinline__ void attendTiles(const TileSmem<HD, Q8> &sm, const void *kHead, const void *vHead, const __half *kSc,
                                            const __half *vSc, uint32_t row0, uint32_t n, uint32_t r0, uint32_t r1, RowOf rowOf = {}) {
    constexpr int DPL = HD / 32, RP = TileSmem<HD, Q8>::kRowPad;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t t0 = 0; t0 < n; t0 += kTile) {
        const uint32_t len = min((uint32_t)kTile, n - t0);
        const auto tileRow = rowOf.tile(row0 + t0, len);
        __syncthreads();   // the previous tile (and the caller's initialisation) is complete
        if constexpr (Q8) {
            for (uint32_t i = threadIdx.x; i < kTile * (HD / 4); i += blockDim.x) {
                const uint32_t rr = i / (HD / 4), c = i % (HD / 4);
                float kf[4] = {0.f, 0.f, 0.f, 0.f}, vf[4] = {0.f, 0.f, 0.f, 0.f};
                if (rr < len) {
                    const size_t off = (size_t)tileRow(row0 + t0 + rr) * HD + 4 * c;
                    loadKv<4, true>(kHead, kSc, off, kf);
                    loadKv<4, true>(vHead, vSc, off, vf);
                }
#pragma unroll
                for (int x = 0; x < 4; x++) { sm.k[rr * RP + 4 * c + x] = kf[x]; sm.v[rr * RP + 4 * c + x] = vf[x]; }
            }
        } else {
            for (uint32_t i = threadIdx.x; i < kTile * (HD / 2); i += blockDim.x) {
                const uint32_t rr = i / (HD / 2), c = i % (HD / 2);
                __nv_bfloat162 kv = __floats2bfloat162_rn(0.f, 0.f), vv = kv;
                if (rr < len) {
                    const size_t off = (size_t)tileRow(row0 + t0 + rr) * HD + 2 * c;
                    kv = *reinterpret_cast<const __nv_bfloat162 *>(reinterpret_cast<const __nv_bfloat16 *>(kHead) + off);
                    vv = *reinterpret_cast<const __nv_bfloat162 *>(reinterpret_cast<const __nv_bfloat16 *>(vHead) + off);
                }
                reinterpret_cast<__nv_bfloat162 *>(sm.k + rr * RP)[c] = kv;
                reinterpret_cast<__nv_bfloat162 *>(sm.v + rr * RP)[c] = vv;
            }
        }
        __syncthreads();
        for (uint32_t r = r0 + warp; r < r1; r += 4) {
            const float *q = sm.q + (size_t)r * HD;
            float s = 0.f;
            if constexpr (Q8) {
                const float *kr = sm.k + lane * RP;
#pragma unroll 8
                for (int c = 0; c < HD / 2; c++) s += q[2 * c] * kr[2 * c] + q[2 * c + 1] * kr[2 * c + 1];
            } else {
                const __nv_bfloat162 *kr = reinterpret_cast<const __nv_bfloat162 *>(sm.k + lane * RP);
#pragma unroll 8
                for (int c = 0; c < HD / 2; c++) {
                    const float2 k2 = __bfloat1622float2(kr[c]);
                    s += q[2 * c] * k2.x + q[2 * c + 1] * k2.y;
                }
            }
            const bool valid = (uint32_t)lane < len;
            const float mOld = sm.m[r];
            const float mNew = fmaxf(mOld, warpMax(valid ? s : -INFINITY));
            const float corr = __expf(mOld - mNew);
            const float pr = valid ? __expf(s - mNew) : 0.f;
            const float lSum = warpSum(pr);
            float acc[DPL];
#pragma unroll
            for (int i = 0; i < DPL; i++) acc[i] = sm.acc[(size_t)r * HD + lane * DPL + i] * corr;
            for (uint32_t u = 0; u < len; u++) {
                const float pu = __shfl_sync(0xffffffffu, pr, u);
                if constexpr (Q8) {
                    const float *vr = sm.v + u * RP + lane * DPL;
#pragma unroll
                    for (int i = 0; i < DPL; i++) acc[i] += pu * vr[i];
                } else {
                    const __nv_bfloat16 *vr = sm.v + u * RP + lane * DPL;
#pragma unroll
                    for (int i = 0; i < DPL; i += 2) {
                        const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(vr + i));
                        acc[i] += pu * v2.x;
                        acc[i + 1] += pu * v2.y;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < DPL; i++) sm.acc[(size_t)r * HD + lane * DPL + i] = acc[i];
            __syncwarp();
            if (lane == 0) { sm.l[r] = sm.l[r] * corr + lSum; sm.m[r] = mNew; }
            __syncwarp();
        }
    }
}

// Launches a tile kernel with `smem` bytes of dynamic shared memory, raising the kernel's limit when a launch needs more than before.
template <auto Kernel, typename Args>
int launchTiles(dim3 grid, size_t smem, cudaStream_t stream, bool pdl, const Args &a) {
    static size_t configured = 0;
    if (smem > configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    DL_CUDA_CHECK(launchPdl(Kernel, grid, dim3(128), smem, stream, pdl, a));
    return 0;
}

}  // namespace

// ---- GEMV-path batch: grid (nHeads, nSplits, nb), block 128 (4 warps). HD in {64, 128} --------------------------------------------
// Every one of the nSplits splits runs, those past nPos empty, so the merge sums the same splits whatever the length.
template <int HD, bool Q8>
__global__ void __launch_bounds__(128) attnDecodeKernel(AttnArgs a) {
    constexpr int DPL = HD / 32;   // dims per lane
    pdlLaunchDependents();
    pdlWait();
    const uint32_t h = blockIdx.x, split = blockIdx.y, t = blockIdx.z;
    const int lane = threadIdx.x & 31;
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
    const size_t headOff = (size_t)kvh * a.seqLen * HD;
    const __half *kSc = Q8 ? a.kScale + headOff / 32 : nullptr, *vSc = Q8 ? a.vScale + headOff / 32 : nullptr;

    float m = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) acc[i] = 0.f;
    scanRows<HD, Q8>(kvPlane<Q8>(a.kCache, headOff), kvPlane<Q8>(a.vCache, headOff), kSc, vSc, q, begin, end, m, l, acc);
    float num, L;
    const float M = combineWarps<HD, false>(m, l, acc, num, L);
    finishSplit<HD>(a.partial, a.counters, (size_t)t * a.nHeads + h, a.nSplits, 1, split, a.nSplits, [&](uint32_t) { return num; },
                    [&](uint32_t) { return make_float2(M, L); }, [&](uint32_t i, float v) {
                        const size_t o = (size_t)t * a.outStride + (size_t)h * HD + i;
                        if (a.outBf16) a.outBf16[o] = __float2bfloat16_rn(v);
                        else a.out[o] = v;
                    });
}

// ---- fused single-token attention: QK-norm + RoPE + KV append + split-KV attention + merge --------------------
// grid (nHeads, nSplits), block 128. The number of *effective* splits is derived from the position on the device
// (effectiveSplit), so short contexts run as one CTA per head with no merge pass at all.
// The current token's K/V never round-trips through the cache: the split that covers position `pos` rotates k
// in registers; the first q-head of every KV group also appends k/v to the cache for later steps.
template <int HD, bool Q8>
__global__ void __launch_bounds__(128) attnFusedKernel(AttnFusedArgs a) {
    constexpr int DPL = HD / 32;
    static_assert(DPL == 2 || DPL == 4, "head dim must be 64 or 128");
    traceStamp(a.trace, 0);
    pdlLaunchDependents();
    pdlWait();
    traceStamp(a.trace, 1);
    const uint32_t h = blockIdx.x, split = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t kvMul = a.nHeads / a.nKvHeads, kvh = h / kvMul;
    int p = a.pos[0];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.seqLen) p = a.seqLen - 1;
    const uint32_t nPos = (uint32_t)p + 1;
    const SplitRange sp = effectiveSplit(nPos, a.nSplits, split);
    if (split >= sp.eff) return;
    const bool ownsNew = sp.end == nPos;                       // this split covers the token being generated
    const uint32_t cachedEnd = ownsNew ? sp.end - 1 : sp.end;  // positions read from the cache: [begin, cachedEnd)

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

    const size_t headOff = (size_t)kvh * a.seqLen * HD;
    void *kHead = kvPlane<Q8>(a.kCache, headOff), *vHead = kvPlane<Q8>(a.vCache, headOff);
    __half *kSc = Q8 ? a.kScale + headOff / 32 : nullptr, *vSc = Q8 ? a.vScale + headOff / 32 : nullptr;
    if (ownsNew && warp == 0) {
        float kn[DPL], vn[DPL];
#pragma unroll
        for (int i = 0; i < DPL; i++) {
            kn[i] = a.qkv[qDim + (size_t)kvh * HD + lane * DPL + i];
            vn[i] = a.qkv[qDim + kvDim + (size_t)kvh * HD + lane * DPL + i];
        }
        normRope(kn, a.kNorm);
        // use the values as the cache stores them here too, so this step matches what later steps will read
        const size_t e = (size_t)p * HD + lane * DPL;
        roundStoreKv<DPL, Q8>(kn, kHead, kSc, e, h % kvMul == 0);
        roundStoreKv<DPL, Q8>(vn, vHead, vSc, e, h % kvMul == 0);
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < DPL; i++) d += q[i] * kn[i];
        d = warpSum(d);
        m = d; l = 1.f;
#pragma unroll
        for (int i = 0; i < DPL; i++) acc[i] = vn[i];
    }

    scanRows<HD, Q8>(kHead, vHead, kSc, vSc, q, sp.begin, cachedEnd, m, l, acc);
    float num, L;
    const float M = combineWarps<HD, true>(m, l, acc, num, L);
    float *outRow = a.out + (size_t)h * HD;
    if (sp.eff == 1) {
        if (threadIdx.x < HD) outRow[threadIdx.x] = num / L;
        traceStamp(a.trace, 3);
        return;
    }
    // finishSplit's protocol written out for one row per CTA. This merge sits on the critical path of every token of the
    // multi-kernel decode path, and the generic row loops measurably slow it at contexts that split. Keep the two in step.
    __shared__ bool sLast;
    float *pOut = a.partial + ((size_t)h * a.nSplits + split) * (HD + 2);
    if (threadIdx.x < HD) pOut[threadIdx.x] = num;
    if (threadIdx.x == 0) { pOut[HD] = M; pOut[HD + 1] = L; }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&a.counters[h], 1u);
        sLast = (prev == sp.eff - 1);
        if (sLast) a.counters[h] = 0;
    }
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    const float *pIn = a.partial + (size_t)h * a.nSplits * (HD + 2);
    float gM = -INFINITY;
    for (uint32_t s = 0; s < sp.eff; s++) gM = fmaxf(gM, __ldcg(pIn + (size_t)s * (HD + 2) + HD));
    if (threadIdx.x < HD) {
        float n2 = 0.f, den = 0.f;
        for (uint32_t s = 0; s < sp.eff; s++) {
            const float ms = __ldcg(pIn + (size_t)s * (HD + 2) + HD);
            const float w = __expf(ms - gM);
            n2 += w * __ldcg(pIn + (size_t)s * (HD + 2) + threadIdx.x);
            den += w * __ldcg(pIn + (size_t)s * (HD + 2) + HD + 1);
        }
        outRow[threadIdx.x] = n2 / den;
    }
}

// ---- choices step: grid (nKvHeads, nSplits), block 128 (4 warps) ------------------------------------------------------------------
// CTA (kvh, split) runs every query row of the KV head over its prefix chunk: R = B * kvMul rows, row r = b * kvMul + g is q-head
// kvh * kvMul + g of choice b. The last effective split also attends each active choice to its own rows.
template <int HD, bool Q8>
__global__ void __launch_bounds__(128) choiceAttnKernel(ChoiceAttnArgs a) {
    pdlLaunchDependents();
    pdlWait();
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t kvMul = a.nHeads / a.nKvHeads, R = a.B * kvMul;
    const TileSmem<HD, Q8> sm(smem, R);
    const uint32_t kvh = blockIdx.x, split = blockIdx.y;
    const SplitRange sp = effectiveSplit(a.P + 1, a.nSplits, split);
    if (split >= sp.eff) return;

    const float scale = rsqrtf((float)HD);
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) {
        const uint32_t r = i / HD, d = i % HD, b = r / kvMul, h = kvh * kvMul + r % kvMul;
        sm.q[i] = a.qkv[(size_t)b * a.qkvStride + (size_t)h * HD + d] * scale;
        sm.acc[i] = 0.f;
    }
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { sm.m[r] = -INFINITY; sm.l[r] = 0.f; }

    const size_t headOff = (size_t)kvh * a.seqLen * HD;
    const void *kHead = kvPlane<Q8>(a.kCache, headOff), *vHead = kvPlane<Q8>(a.vCache, headOff);
    const __half *kSc = Q8 ? a.kScale + headOff / 32 : nullptr, *vSc = Q8 ? a.vScale + headOff / 32 : nullptr;
    attendTiles(sm, kHead, vHead, kSc, vSc, sp.begin, sp.end - sp.begin, 0, R);
    if (split == sp.eff - 1) {
        for (uint32_t b = 0; b < a.B; b++) {
            if ((a.inactiveMask >> b) & 1u) continue;
            attendTiles(sm, kHead, vHead, kSc, vSc, a.P + 1 + b * a.C, a.j + 1, b * kvMul, (b + 1) * kvMul);
        }
    }
    __syncthreads();

    auto store = [&](uint32_t i, float v) {
        const uint32_t r = i / HD, d = i % HD, b = r / kvMul, h = kvh * kvMul + r % kvMul;
        a.out[(size_t)b * a.outStride + (size_t)h * HD + d] = v;
    };
    if (sp.eff == 1) {
        for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) store(i, sm.acc[i] / sm.l[i / HD]);
        return;
    }
    finishSplit<HD>(a.partial, a.counters, kvh, a.nSplits, R, split, sp.eff,
                    [&](uint32_t i) { return sm.acc[i]; }, [&](uint32_t r) { return make_float2(sm.m[r], sm.l[r]); }, store);
}

// ---- slots step: grid (nKvHeads, nSplits, B), block 128 (4 warps) -----------------------------------------------------------------
// CTA (kvh, split, b) runs the kvMul q-heads of the KV head over its chunk of row b's slot (one q-head per warp, round robin).
// PAGED: the slot's rows are read through its page table from planes of planeRows rows per KV head; the tiles and splits are those
// of the contiguous slot.
template <int HD, bool Q8, bool PAGED>
__global__ void __launch_bounds__(128) slotAttnKernel(typename std::conditional<PAGED, PagedSlotAttnArgs, SlotAttnArgs>::type a) {
    pdlLaunchDependents();
    pdlWait();
    const uint32_t kvh = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
    if (b < 32 && ((a.inactiveMask >> b) & 1u)) return;
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t R = a.nHeads / a.nKvHeads;   // q-heads of this KV head
    const TileSmem<HD, Q8> sm(smem, R);
    int p = a.pos[b];
    if (p < 0) p = 0;
    if ((uint32_t)p >= a.L) p = (int)a.L - 1;
    const SplitRange sp = effectiveSplit((uint32_t)p + 1, a.nSplits, split);
    if (split >= sp.eff) return;

    const float scale = rsqrtf((float)HD);
    const float *qRow = a.qkv + (size_t)b * a.qkvStride + (size_t)kvh * R * HD;
    for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) { sm.q[i] = qRow[i] * scale; sm.acc[i] = 0.f; }
    for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) { sm.m[r] = -INFINITY; sm.l[r] = 0.f; }

    if constexpr (PAGED) {
        const size_t headOff = (size_t)kvh * a.planeRows * HD;
        attendTiles(sm, kvPlane<Q8>(a.kCache, headOff), kvPlane<Q8>(a.vCache, headOff), Q8 ? a.kScale + headOff / 32 : nullptr,
                    Q8 ? a.vScale + headOff / 32 : nullptr, sp.begin, sp.end - sp.begin, 0, R, PagedRows{a.pageTable + (size_t)b * a.pageStride});
    } else {
        const size_t headOff = (size_t)b * a.slotStride + (size_t)kvh * a.L * HD;
        attendTiles(sm, kvPlane<Q8>(a.kCache, headOff), kvPlane<Q8>(a.vCache, headOff), Q8 ? a.kScale + headOff / 32 : nullptr,
                    Q8 ? a.vScale + headOff / 32 : nullptr, sp.begin, sp.end - sp.begin, 0, R);
    }
    __syncthreads();

    float *outRow = a.out + (size_t)b * a.outStride + (size_t)kvh * R * HD;
    if (sp.eff == 1) {
        for (uint32_t i = threadIdx.x; i < R * HD; i += blockDim.x) outRow[i] = sm.acc[i] / sm.l[i / HD];
        return;
    }
    finishSplit<HD>(a.partial, a.counters, (size_t)b * a.nKvHeads + kvh, a.nSplits, R, split, sp.eff,
                    [&](uint32_t i) { return sm.acc[i]; }, [&](uint32_t r) { return make_float2(sm.m[r], sm.l[r]); },
                    [&](uint32_t i, float v) { outRow[i] = v; });
}

int launchAttnDecode(const AttnArgs &a, int nb, cudaStream_t stream, bool pdl) {
    const dim3 grid(a.nHeads, a.nSplits, nb);
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    const bool q8 = a.kScale != nullptr;
    if (a.headDim == 128) DL_CUDA_CHECK(launchPdl(q8 ? attnDecodeKernel<128, true> : attnDecodeKernel<128, false>, grid, dim3(128), 0, stream, pdl, a));
    else if (a.headDim == 64) DL_CUDA_CHECK(launchPdl(q8 ? attnDecodeKernel<64, true> : attnDecodeKernel<64, false>, grid, dim3(128), 0, stream, pdl, a));
    else return -1;
    return 0;
}

int launchAttnFused(const AttnFusedArgs &a, cudaStream_t stream, bool pdl) {
    const dim3 grid(a.nHeads, a.nSplits);
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    const bool q8 = a.kScale != nullptr;
    if (a.headDim == 128) DL_CUDA_CHECK(launchPdl(q8 ? attnFusedKernel<128, true> : attnFusedKernel<128, false>, grid, dim3(128), 0, stream, pdl, a));
    else if (a.headDim == 64) DL_CUDA_CHECK(launchPdl(q8 ? attnFusedKernel<64, true> : attnFusedKernel<64, false>, grid, dim3(128), 0, stream, pdl, a));
    else return -1;
    return 0;
}

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
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    const uint32_t R = a.B * (a.nHeads / a.nKvHeads);
    const dim3 grid(a.nKvHeads, a.nSplits);
    if (a.kScale) {
        if (a.headDim == 128) return launchTiles<choiceAttnKernel<128, true>>(grid, TileSmem<128, true>::bytes(R), stream, pdl, a);
        if (a.headDim == 64) return launchTiles<choiceAttnKernel<64, true>>(grid, TileSmem<64, true>::bytes(R), stream, pdl, a);
        return -1;
    }
    if (a.headDim == 128) return launchTiles<choiceAttnKernel<128, false>>(grid, TileSmem<128, false>::bytes(R), stream, pdl, a);
    if (a.headDim == 64) return launchTiles<choiceAttnKernel<64, false>>(grid, TileSmem<64, false>::bytes(R), stream, pdl, a);
    return -1;
}

template <bool PAGED, typename Args>
static int launchSlotAttnAs(const Args &a, cudaStream_t stream, bool pdl) {
    if (a.nKvHeads == 0 || a.nHeads % a.nKvHeads || a.nSplits < 1 || a.L < 1 || a.B < 1 || a.B > 32) return -1;
    if ((a.kScale == nullptr) != (a.vScale == nullptr)) return -1;
    const uint32_t R = a.nHeads / a.nKvHeads;
    const dim3 grid(a.nKvHeads, a.nSplits, a.B);
    if (a.kScale) {
        if (a.headDim == 128) return launchTiles<slotAttnKernel<128, true, PAGED>>(grid, TileSmem<128, true>::bytes(R), stream, pdl, a);
        if (a.headDim == 64) return launchTiles<slotAttnKernel<64, true, PAGED>>(grid, TileSmem<64, true>::bytes(R), stream, pdl, a);
        return -1;
    }
    if (a.headDim == 128) return launchTiles<slotAttnKernel<128, false, PAGED>>(grid, TileSmem<128, false>::bytes(R), stream, pdl, a);
    if (a.headDim == 64) return launchTiles<slotAttnKernel<64, false, PAGED>>(grid, TileSmem<64, false>::bytes(R), stream, pdl, a);
    return -1;
}

int launchSlotAttn(const SlotAttnArgs &a, cudaStream_t stream, bool pdl) { return launchSlotAttnAs<false>(a, stream, pdl); }

int launchSlotAttnPaged(const PagedSlotAttnArgs &a, cudaStream_t stream, bool pdl) {
    if (!a.pageTable || a.pageStride < (a.L + kPageRows - 1) / kPageRows || a.planeRows < a.L) return -1;
    return launchSlotAttnAs<true>(a, stream, pdl);
}

}  // namespace dl

// Stand-alone entry points for the unit tests and measurements (tests/test_gpu_decode_attn.py, test_gpu_choices.py,
// test_gpu_slots.py, tools/bench_*.py): each fills the argument struct and calls the launcher without programmatic dependent launch.
// Pointers are device pointers; caches are bf16 [nKvHeads][seqLen][headDim].
DL_EXPORT int dl_attn_decode(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, uint32_t nHeads,
                             uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits, float *partial, unsigned int *counters,
                             float *out, uint32_t outStride, void *outBf16, int nb, cudaStream_t stream) {
    dl::AttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos;
    a.kCache = kCache; a.vCache = vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride; a.outBf16 = (__nv_bfloat16 *)outBf16;
    return dl::launchAttnDecode(a, nb, stream, false);
}

DL_EXPORT int dl_attn_fused(const float *qkv, const int *pos, const float *rope, const float *qNorm, const float *kNorm, float eps,
                            void *kCache, void *vCache, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen,
                            uint32_t nSplits, float *partial, unsigned int *counters, float *out, cudaStream_t stream) {
    dl::AttnFusedArgs a{};
    a.qkv = qkv; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.kCache = kCache; a.vCache = vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out;
    return dl::launchAttnFused(a, stream, false);
}

// QK-norm + RoPE of B query rows at rotary position P + 1 + j, K/V append of the active rows at P + 1 + b * C + j (ropeKvKernel),
// then choiceAttnKernel. Every row of `pos` (device, [B]) must hold P + 1 + j.
DL_EXPORT int dl_choice_attn(float *qkv, uint32_t qkvStride, const int *pos, const float *rope, const float *qNorm, const float *kNorm, float eps,
                             void *kCache, void *vCache, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits,
                             uint32_t B, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, float *partial, unsigned int *counters,
                             float *out, uint32_t outStride, cudaStream_t stream) {
    dl::RopeKvArgs r{};
    r.qkv = qkv; r.qkvStride = qkvStride; r.pos = pos; r.rope = rope; r.qNorm = qNorm; r.kNorm = kNorm; r.eps = eps;
    r.nHeads = nHeads; r.nKvHeads = nKvHeads; r.headDim = headDim; r.seqLen = seqLen;
    r.kCache = kCache; r.vCache = vCache; r.rowStride = C; r.inactiveMask = inactiveMask;
    dl::ChoiceAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.kCache = r.kCache; a.vCache = r.vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.B = B; a.P = P; a.C = C; a.j = j; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    if (!dl::choiceRowsFit(B, P, C, j, inactiveMask, seqLen)) return -1;   // before anything is written
    const int rc = dl::launchRopeKv(r, (int)B, stream, false);
    if (rc != 0) return rc;
    return dl::launchChoiceAttn(a, stream, false);
}

// choiceAttnKernel alone over q rows that are already normalised and rotated, with the choices' K/V rows already in the cache.
DL_EXPORT int dl_choice_attn_only(const float *qkv, uint32_t qkvStride, const void *kCache, const void *vCache, uint32_t nHeads, uint32_t nKvHeads,
                                  uint32_t headDim, uint32_t seqLen, uint32_t nSplits, uint32_t B, uint32_t P, uint32_t C, uint32_t j,
                                  uint32_t inactiveMask, float *partial, unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::ChoiceAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.kCache = kCache; a.vCache = vCache;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.B = B; a.P = P; a.C = C; a.j = j; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchChoiceAttn(a, stream, false);
}

// slotAttnKernel alone over q rows that are already normalised and rotated, with every row's K/V already in its slot. pos is a
// device [B] array.
DL_EXPORT int dl_slot_attn(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, uint32_t nHeads,
                           uint32_t nKvHeads, uint32_t headDim, uint32_t L, uint32_t nSplits, uint32_t B, uint32_t inactiveMask, float *partial,
                           unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::SlotAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.kCache = kCache; a.vCache = vCache;
    a.slotStride = (uint64_t)nKvHeads * L * headDim; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.L = L;
    a.nSplits = nSplits; a.B = B; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchSlotAttn(a, stream, false);
}

// q80 variants of the entry points above: kCache / vCache are the int8 value planes, kScale / vScale the f16 scale planes
// [nKvHeads][seqLen][headDim / 32] (for slots: every slot's, at element offset slot * slotStride / 32).
DL_EXPORT int dl_attn_decode_q80(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, const void *kScale,
                                 const void *vScale, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits,
                                 float *partial, unsigned int *counters, float *out, uint32_t outStride, void *outBf16, int nb, cudaStream_t stream) {
    dl::AttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos;
    a.kCache = kCache; a.vCache = vCache; a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride; a.outBf16 = (__nv_bfloat16 *)outBf16;
    return dl::launchAttnDecode(a, nb, stream, false);
}

DL_EXPORT int dl_attn_fused_q80(const float *qkv, const int *pos, const float *rope, const float *qNorm, const float *kNorm, float eps,
                                void *kCache, void *vCache, void *kScale, void *vScale, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim,
                                uint32_t seqLen, uint32_t nSplits, float *partial, unsigned int *counters, float *out, cudaStream_t stream) {
    dl::AttnFusedArgs a{};
    a.qkv = qkv; a.pos = pos; a.rope = rope; a.qNorm = qNorm; a.kNorm = kNorm; a.eps = eps;
    a.kCache = kCache; a.vCache = vCache; a.kScale = (__half *)kScale; a.vScale = (__half *)vScale;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.partial = partial; a.counters = counters; a.out = out;
    return dl::launchAttnFused(a, stream, false);
}

DL_EXPORT int dl_choice_attn_only_q80(const float *qkv, uint32_t qkvStride, const void *kCache, const void *vCache, const void *kScale,
                                      const void *vScale, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t seqLen, uint32_t nSplits,
                                      uint32_t B, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, float *partial, unsigned int *counters,
                                      float *out, uint32_t outStride, cudaStream_t stream) {
    dl::ChoiceAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.kCache = kCache; a.vCache = vCache; a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.seqLen = seqLen; a.nSplits = nSplits;
    a.B = B; a.P = P; a.C = C; a.j = j; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchChoiceAttn(a, stream, false);
}

DL_EXPORT int dl_slot_attn_q80(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, const void *kScale,
                               const void *vScale, uint32_t nHeads, uint32_t nKvHeads, uint32_t headDim, uint32_t L, uint32_t nSplits, uint32_t B,
                               uint32_t inactiveMask, float *partial, unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::SlotAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.kCache = kCache; a.vCache = vCache;
    a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale;
    a.slotStride = (uint64_t)nKvHeads * L * headDim; a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.L = L;
    a.nSplits = nSplits; a.B = B; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchSlotAttn(a, stream, false);
}

// slotAttnKernel over paged slots (tests/test_gpu_paged_slots.py): the planes hold planeRows rows per KV head, row b's logical row r
// is at physical row pageTable[b * pageStride + r / 64] * 64 + r % 64 (pageTable: device int32). kScale / vScale null: bf16 planes.
DL_EXPORT int dl_slot_attn_paged(const float *qkv, uint32_t qkvStride, const int *pos, const void *kCache, const void *vCache, const void *kScale,
                                 const void *vScale, const int32_t *pageTable, uint32_t pageStride, uint32_t planeRows, uint32_t nHeads,
                                 uint32_t nKvHeads, uint32_t headDim, uint32_t L, uint32_t nSplits, uint32_t B, uint32_t inactiveMask,
                                 float *partial, unsigned int *counters, float *out, uint32_t outStride, cudaStream_t stream) {
    dl::PagedSlotAttnArgs a{};
    a.qkv = qkv; a.qkvStride = qkvStride; a.pos = pos; a.kCache = kCache; a.vCache = vCache;
    a.kScale = (const __half *)kScale; a.vScale = (const __half *)vScale;
    a.pageTable = pageTable; a.pageStride = pageStride; a.planeRows = planeRows;
    a.nHeads = nHeads; a.nKvHeads = nKvHeads; a.headDim = headDim; a.L = L;
    a.nSplits = nSplits; a.B = B; a.inactiveMask = inactiveMask; a.partial = partial; a.counters = counters; a.out = out; a.outStride = outStride;
    return dl::launchSlotAttnPaged(a, stream, false);
}
