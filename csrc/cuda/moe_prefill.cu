// Mixture-of-experts feed-forward over a prompt chunk (T tokens): routing -> token sort by expert -> grouped tensor-core GEMMs ->
// weighted combine (+ tensor/expert-parallel all-reduce over peer memory).
//
// Reference: the MoE branch of buildLlmNet (src/llm.cpp:425-499) run at nBatches = 32: REPEAT_Z, gate MATMUL, SOFTMAX, MOE_GATE, per
// active expert MATMUL w1/w3 + SILU + MUL + MATMUL w2, SCALE, MERGE_SUM (src/nn/nn-cpu-ops.cpp:1138-1192,1462-1492) — one GEMV per
// (token, expert) pair. Here the (token, expert) pairs of the whole chunk are sorted by expert so every expert's weights are read
// once per chunk and multiplied on the tensor cores (gemmQ40TcGrouped): dispatch = a gather into expert-sorted rows, combine = a
// deterministic weighted sum per token in routing-slot order, pushed to every rank through LL words when experts are sharded.
#include <algorithm>

#include "kernels.h"

namespace dl {
namespace {

// One CTA. pairs p = t * k + j (token t, routing slot j). Stable counting sort by expert:
//   count[e], offset[e] (exclusive prefix), slotOfPair[p] = sorted row of pair p, tokenOfSlot[s] = token of sorted row s.
// Experts outside [firstLocal, firstLocal + nLocal) get count 0 (expert parallelism: their pairs are computed on another rank) and
// slotOfPair = -1. Group index in the outputs is the LOCAL expert index (e - firstLocal), matching the rank's weight storage.
__global__ void __launch_bounds__(256) moeSortKernel(const int *__restrict__ expertIdx, uint32_t nPairs, uint32_t k, uint32_t nExperts,
                                                      uint32_t firstLocal, uint32_t nLocal, int *count, int *offset, int *slotOfPair,
                                                      int *tokenOfSlot, int *totalRows) {
    extern __shared__ int sh[];          // [nPairs] expert of every pair, then [nLocal + 1] offsets
    int *sExp = sh, *sOff = sh + nPairs;
    for (uint32_t p = threadIdx.x; p < nPairs; p += blockDim.x) sExp[p] = expertIdx[p];
    __syncthreads();
    // thread g counts the pairs of local expert g
    int myCount = 0;
    const uint32_t g = threadIdx.x;
    if (g < nLocal) {
        const int e = (int)(firstLocal + g);
        for (uint32_t p = 0; p < nPairs; p++) myCount += (sExp[p] == e) ? 1 : 0;
        sOff[g] = myCount;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (uint32_t i = 0; i < nLocal; i++) { const int c = sOff[i]; sOff[i] = run; run += c; }
        sOff[nLocal] = run;
        *totalRows = run;
    }
    __syncthreads();
    if (g < nLocal) {
        const int e = (int)(firstLocal + g);
        count[g] = myCount;
        offset[g] = sOff[g];
        int pos = sOff[g];
        for (uint32_t p = 0; p < nPairs; p++) {
            if (sExp[p] == e) {
                slotOfPair[p] = pos;
                tokenOfSlot[pos] = (int)(p / k);
                pos++;
            }
        }
    }
    for (uint32_t p = threadIdx.x; p < nPairs; p += blockDim.x) {
        const int e = sExp[p];
        if (e < (int)firstLocal || e >= (int)(firstLocal + nLocal)) slotOfPair[p] = -1;
    }
}

// xs[s][:] = xn[tokenOfSlot[s]][:] (bf16 rows, 16 bytes per thread)
__global__ void __launch_bounds__(256) moeGatherKernel(const __nv_bfloat16 *__restrict__ xn, uint32_t dim, const int *__restrict__ tokenOfSlot,
                                                        const int *__restrict__ totalRows, __nv_bfloat16 *__restrict__ xs) {
    const uint32_t s = blockIdx.x;
    if ((int)s >= *totalRows) return;
    const uint4 *src = reinterpret_cast<const uint4 *>(xn + (size_t)tokenOfSlot[s] * dim);
    uint4 *dst = reinterpret_cast<uint4 *>(xs + (size_t)s * dim);
    for (uint32_t i = threadIdx.x; i < dim / 8; i += blockDim.x) dst[i] = src[i];
}

// x[t][f] += sum_j weight[t][j] * ys[slotOfPair[t*k+j]][f]   (pairs with slot -1 contribute nothing on this rank)
// With ar.nRanks > 1 the per-rank partial sums are exchanged through LL words (same protocol as the GEMM + all-reduce epilogue,
// gemm_q40_tc.cu) and summed in rank order before the residual add, so every rank ends with the same x.
__global__ void __launch_bounds__(256) moeCombineKernel(float *x, uint32_t dim, uint32_t T, uint32_t k, const float *__restrict__ ys,
                                                         const int *__restrict__ slotOfPair, const float *__restrict__ weight, ArArgs ar) {
    const uint32_t t = blockIdx.y;
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= dim || t >= T) return;
    float acc = 0.f;
    for (uint32_t j = 0; j < k; j++) {
        const int s = slotOfPair[t * k + j];
        if (s >= 0) acc += weight[t * k + j] * ys[(size_t)s * dim + f];
    }
    if (ar.nRanks > 1) {
        const size_t cell = (size_t)t * ar.dim + f;
        const size_t mineOff = (size_t)(ar.parity * ar.nRanks + ar.rank) * ar.slotStride + cell;
        for (uint32_t p = 0; p < ar.nRanks; p++) stLL(ar.slots[(ar.rank + p) % ar.nRanks] + mineOff, __float_as_uint(acc), 1u);
        float sum = 0.f;
        uint64_t *mine = ar.slots[ar.rank];
        for (uint32_t sr = 0; sr < ar.nRanks; sr++) {
            uint64_t *w = mine + (size_t)(ar.parity * ar.nRanks + sr) * ar.slotStride + cell;
            uint2 v = ldLL(w);
            uint32_t spins = 0;
            while (v.y == 0u && ++spins < (1u << 28)) v = ldLL(w);
            sum += __uint_as_float(v.x);
            stLL(w, 0u, 0u);
        }
        acc = sum;
    }
    x[(size_t)t * dim + f] += acc;
}

// x[t][f] += sum over ranks of partial_r[t][f]: the tensor-parallel all-reduce + residual of a prompt chunk as its own kernel, so
// that the producing GEMM keeps split-K and all SMs (the fused GEMM + all-reduce epilogue pins one CTA per 128-row tile while it
// polls). Push: one multimem.st per cell through the NVSwitch multicast mapping (or nRanks unicast stores); pull: the N source
// slots of the cell, summed in rank order.
__global__ void __launch_bounds__(256) arResidualKernel(float *x, const float *__restrict__ partial, uint32_t dim, uint32_t T, ArArgs ar) {
    pdlLaunchDependents();
    pdlWait();
    const uint32_t t = blockIdx.y;
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= dim || t >= T) return;
    const float mineV = partial[(size_t)t * dim + f];
    const size_t cell = (size_t)t * ar.dim + f;
    const size_t mineOff = (size_t)(ar.parity * ar.nRanks + ar.rank) * ar.slotStride + cell;
    if (ar.slotsMc) {
        const uint64_t word = (uint64_t)__float_as_uint(mineV) | (1ull << 32);
        asm volatile("multimem.st.relaxed.sys.global.b64 [%0], %1;" ::"l"(ar.slotsMc + mineOff), "l"(word) : "memory");
    } else {
        for (uint32_t p = 0; p < ar.nRanks; p++) stLL(ar.slots[(ar.rank + p) % ar.nRanks] + mineOff, __float_as_uint(mineV), 1u);
    }
    float sum = 0.f;
    uint64_t *mine = ar.slots[ar.rank];
    for (uint32_t sr = 0; sr < ar.nRanks; sr++) {
        uint64_t *w = mine + (size_t)(ar.parity * ar.nRanks + sr) * ar.slotStride + cell;
        uint2 v = ldLL(w);
        uint32_t spins = 0;
        while (v.y == 0u && ++spins < (1u << 28)) v = ldLL(w);
        sum += __uint_as_float(v.x);
        stLL(w, 0u, 0u);
    }
    x[(size_t)t * dim + f] += sum;
}

struct MoeScratch {
    int *count = nullptr, *offset = nullptr, *slotOfPair = nullptr, *tokenOfSlot = nullptr, *totalRows = nullptr;
    int *expertIdx = nullptr;
    float *expertWeight = nullptr, *routerLogits = nullptr;
    unsigned int *routerCounter = nullptr;
    __nv_bfloat16 *xs = nullptr, *hs = nullptr;
    float *ys = nullptr;
    size_t capPairs = 0, capDim = 0, capFf = 0, capExperts = 0, capTokens = 0;
    uint32_t lastT = 0, lastK = 0, lastExperts = 0, lastFf = 0;   // shape of the call whose data the scratch holds (moePrefillScratchRead)
};
MoeScratch gMoe;

// The router scratch is [T][nExperts] logits + [T] counters, so the token count is a capacity of its own: a chunk with more
// tokens but fewer pairs per token (smaller k) than an earlier one must still reallocate. Capacities only grow.
int moeEnsureScratch(uint32_t nPairs, uint32_t dim, uint32_t ff, uint32_t nExperts, uint32_t T) {
    MoeScratch &m = gMoe;
    if (nPairs <= m.capPairs && dim <= m.capDim && ff <= m.capFf && nExperts <= m.capExperts && T <= m.capTokens) return 0;
    nPairs = std::max(nPairs, (uint32_t)m.capPairs); dim = std::max(dim, (uint32_t)m.capDim); ff = std::max(ff, (uint32_t)m.capFf);
    nExperts = std::max(nExperts, (uint32_t)m.capExperts); T = std::max(T, (uint32_t)m.capTokens);
    for (void *p : {(void *)m.count, (void *)m.offset, (void *)m.slotOfPair, (void *)m.tokenOfSlot, (void *)m.totalRows, (void *)m.expertIdx,
                    (void *)m.expertWeight, (void *)m.routerLogits, (void *)m.routerCounter, (void *)m.xs, (void *)m.hs, (void *)m.ys})
        if (p) cudaFree(p);
    m = MoeScratch{};
    const size_t P = nPairs, E = nExperts;
    DL_CUDA_CHECK(cudaMalloc(&m.count, (E + 1) * 4)); DL_CUDA_CHECK(cudaMalloc(&m.offset, (E + 1) * 4));
    DL_CUDA_CHECK(cudaMalloc(&m.slotOfPair, P * 4)); DL_CUDA_CHECK(cudaMalloc(&m.tokenOfSlot, P * 4)); DL_CUDA_CHECK(cudaMalloc(&m.totalRows, 64));
    DL_CUDA_CHECK(cudaMalloc(&m.expertIdx, P * 4)); DL_CUDA_CHECK(cudaMalloc(&m.expertWeight, P * 4));
    DL_CUDA_CHECK(cudaMalloc(&m.routerLogits, (size_t)T * E * 4)); DL_CUDA_CHECK(cudaMalloc(&m.routerCounter, (size_t)T * 4));
    DL_CUDA_CHECK(cudaMemset(m.routerCounter, 0, (size_t)T * 4));
    // activation rows carry a tail of 256 zero rows: the grouped GEMM's TMA boxes read up to nTile rows past a group's first row
    DL_CUDA_CHECK(cudaMalloc(&m.xs, (P + 256) * dim * 2)); DL_CUDA_CHECK(cudaMemset(m.xs, 0, (P + 256) * dim * 2));
    DL_CUDA_CHECK(cudaMalloc(&m.hs, (P + 256) * ff * 2)); DL_CUDA_CHECK(cudaMemset(m.hs, 0, (P + 256) * ff * 2));
    DL_CUDA_CHECK(cudaMalloc(&m.ys, P * dim * 4));
    m.capPairs = nPairs; m.capDim = dim; m.capFf = ff; m.capExperts = nExperts; m.capTokens = T;
    return 0;
}

// out[p][:] = hs[slotOfPair[p]][:] (bf16 rows in pair order; a pair of another rank's expert gets zeros)
__global__ void __launch_bounds__(256) moePairRowsKernel(const __nv_bfloat16 *__restrict__ hs, uint32_t ff, const int *__restrict__ slotOfPair,
                                                          __nv_bfloat16 *__restrict__ out) {
    const uint32_t p = blockIdx.x;
    const int s = slotOfPair[p];
    for (uint32_t i = threadIdx.x; i < ff; i += blockDim.x)
        out[(size_t)p * ff + i] = s >= 0 ? hs[(size_t)s * ff + i] : __float2bfloat16(0.f);
}

}  // namespace

// What the last moePrefillFfn call of the process left in its scratch, for T tokens of k routing slots (tests): router logits
// [T][nExperts] f32, expert ids and weights [T][k], and the SwiGLU output of every (token, slot) pair [T][k][ff] bf16 in pair order.
// A null destination is skipped; -1 unless the last call had exactly this T, k, nExperts and ff.
int moePrefillScratchRead(uint32_t T, uint32_t k, uint32_t nExperts, uint32_t ff, float *logits, int *ids, float *weights,
                          __nv_bfloat16 *hPairs, cudaStream_t stream) {
    const MoeScratch &m = gMoe;
    if (T == 0 || T != m.lastT || k != m.lastK || nExperts != m.lastExperts || ff != m.lastFf) return -1;
    if (logits) DL_CUDA_CHECK(cudaMemcpyAsync(logits, m.routerLogits, (size_t)T * nExperts * 4, cudaMemcpyDeviceToDevice, stream));
    if (ids) DL_CUDA_CHECK(cudaMemcpyAsync(ids, m.expertIdx, (size_t)T * k * 4, cudaMemcpyDeviceToDevice, stream));
    if (weights) DL_CUDA_CHECK(cudaMemcpyAsync(weights, m.expertWeight, (size_t)T * k * 4, cudaMemcpyDeviceToDevice, stream));
    if (hPairs) {
        moePairRowsKernel<<<T * k, 256, 0, stream>>>(m.hs, ff, m.slotOfPair, hPairs);
        DL_CUDA_CHECK(cudaGetLastError());
    }
    return 0;
}

int launchArResidual(float *x, const float *partial, uint32_t dim, uint32_t T, const ArArgs &ar, cudaStream_t stream, bool pdl) {
    DL_CUDA_CHECK(launchPdl(arResidualKernel, dim3((dim + 255) / 256, T), dim3(256), 0, stream, pdl, x, partial, dim, T, ar));
    return 0;
}

// MoE feed-forward of a prompt chunk: x [T][dim] f32 (residual stream, updated in place), xnScratch bf16 [T][dim].
// w13: [nLocal][2*ff][dim] gate/up interleaved, w2: [nLocal][dim][ff]. Returns 1 when the shape is not covered by the grouped GEMM.
int moePrefillFfn(const MoePrefillArgs &a, cudaStream_t stream) {
    const uint32_t nPairs = a.T * a.k;
    if (a.T == 0 || a.T > 256 || a.nLocal > 256 || a.nExperts > 256 || a.dim % 256 || a.ff % 256 || a.dim % 8) return 1;
    if (nPairs * 4 + (a.nLocal + 1) * 4 > 40 * 1024) return 1;
    { const int r = moeEnsureScratch(nPairs, a.dim, a.ff, a.nExperts, a.T); if (r != 0) return r; }
    MoeScratch &m = gMoe;
    m.lastT = a.T; m.lastK = a.k; m.lastExperts = a.nExperts; m.lastFf = a.ff;
    RouterArgs ro{};
    ro.x = a.x; ro.normW = a.norm; ro.gate = a.gate; ro.eps = a.eps; ro.dim = a.dim; ro.nExperts = a.nExperts; ro.k = a.k;
    ro.logits = m.routerLogits; ro.counter = m.routerCounter; ro.expertIdx = m.expertIdx; ro.expertWeight = m.expertWeight;
    { const int r = launchMoeRouter(ro, (int)a.T, stream, false); if (r != 0) return r; }
    moeSortKernel<<<1, 256, nPairs * 4 + (a.nLocal + 1) * 4, stream>>>(m.expertIdx, nPairs, a.k, a.nExperts, a.firstLocal, a.nLocal, m.count, m.offset,
                                                                        m.slotOfPair, m.tokenOfSlot, m.totalRows);
    DL_CUDA_CHECK(cudaGetLastError());
    { const int r = launchRmsNormBf16(a.x, a.dim, a.norm, a.xnScratch, a.dim, a.dim, a.eps, a.T, stream); if (r != 0) return r; }
    moeGatherKernel<<<nPairs, 256, 0, stream>>>((const __nv_bfloat16 *)a.xnScratch, a.dim, m.tokenOfSlot, m.totalRows, m.xs);
    DL_CUDA_CHECK(cudaGetLastError());
    { const int r = gemmQ40TcGrouped(GEPI_SWIGLU_BF16_, a.w13Qs, a.w13Sc, a.nLocal, 2 * a.ff, a.dim, m.xs, a.dim, nPairs + 256, a.T, m.count, m.offset,
                                     m.hs, a.ff, a.numSms, stream); if (r != 0) return r; }
    { const int r = gemmQ40TcGrouped(GEPI_STORE_F32_, a.w2Qs, a.w2Sc, a.nLocal, a.dim, a.ff, m.hs, a.ff, nPairs + 256, a.T, m.count, m.offset,
                                     m.ys, a.dim, a.numSms, stream); if (r != 0) return r; }
    moeCombineKernel<<<dim3((a.dim + 255) / 256, a.T), 256, 0, stream>>>(a.x, a.dim, a.T, a.k, m.ys, m.slotOfPair, m.expertWeight, a.ar);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace dl

// Stand-alone entry point for the unit tests (tests/test_gpu_moe.py): moePrefillFfn on one rank, with the gate activation passed
// explicitly (0 = SiLU, 1 = GELU) instead of the one of the last engine created. The routing the call used (expert id and weight
// of every pair, [T][k]) is copied to expertIdxOut / expertWeightOut.
DL_EXPORT int dl_moe_prefill_ffn(float *x, void *xnScratch, const float *norm, const float *gate, const void *w13Qs, const void *w13Sc,
                                 const void *w2Qs, const void *w2Sc, uint32_t T, uint32_t dim, uint32_t ff, uint32_t nExperts, uint32_t k,
                                 uint32_t firstLocal, uint32_t nLocal, float eps, int numSms, uint32_t hiddenAct, int *expertIdxOut,
                                 float *expertWeightOut, cudaStream_t stream) {
    dl::MoePrefillArgs a{};
    a.x = x; a.xnScratch = xnScratch; a.norm = norm; a.gate = gate; a.w13Qs = w13Qs; a.w13Sc = w13Sc; a.w2Qs = w2Qs; a.w2Sc = w2Sc;
    a.T = T; a.dim = dim; a.ff = ff; a.nExperts = nExperts; a.k = k; a.firstLocal = firstLocal; a.nLocal = nLocal; a.eps = eps; a.numSms = numSms;
    const dl::HiddenActScope act(hiddenAct);
    const int r = dl::moePrefillFfn(a, stream);
    if (r != 0) return r;
    DL_CUDA_CHECK(cudaMemcpyAsync(expertIdxOut, dl::gMoe.expertIdx, (size_t)T * k * sizeof(int), cudaMemcpyDeviceToDevice, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(expertWeightOut, dl::gMoe.expertWeight, (size_t)T * k * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return 0;
}

// The capacities of the MoE prefill scratch (tests): pairs, dim, ff, experts, tokens. They only grow; a call beyond any of them
// reallocates every buffer.
DL_EXPORT void dl_moe_scratch_caps(uint64_t out[5]) {
    const dl::MoeScratch &m = dl::gMoe;
    out[0] = m.capPairs; out[1] = m.capDim; out[2] = m.capFf; out[3] = m.capExperts; out[4] = m.capTokens;
}
