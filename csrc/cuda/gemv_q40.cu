// Decode-path matrix-vector kernels: y[t][d] = W_q40[d][n] · q80(x[t][n]) for 1..8 tokens, fused with the
// element-wise work around them.
//
// Replaces these reference op chains (one launch each instead of 3-6 barrier-separated ops):
//   INV_RMS + RMS_NORM + CAST(f32->q80) + MATMUL(q80×q40)            src/llm.cpp:283-320, :412-423, :567-592
//   CAST(f32->q80) + MATMUL + [all-gather + MERGE_ADD residual]      src/llm.cpp:385-411, :533-566
//   ... + SILU + MUL (SwiGLU)                                        src/llm.cpp:509-532
// The integer math is the reference's Q80×Q40 contract (nn-cpu-ops.cpp:231-449: int8 dot per 32-block, scaled
// by d_w·d_x); everything else about the kernel is specific to the GPU:
//   * one persistent CTA per SM (512 threads); each CTA owns a contiguous, pair-aligned row tile, so the
//     per-SM byte share of the weight stream is equal to within one row pair;
//   * a warp-step = (row, 32-block segment): lanes read 512 contiguous bytes of nibbles, U steps are issued
//     back to back before any math so ~64 KB/SM is in flight;
//   * PDL: the first U steps of weight loads are issued *before* griddepcontrol.wait, i.e. while the producer
//     kernel is still draining — the weight stream never stops at kernel boundaries;
//   * the activation vector is normalised + quantised once per CTA into shared memory in a dp4a-friendly
//     plane layout (conflict-free 16 B reads per lane);
//   * deterministic reduction: per-(row,segment) partials in shared memory, summed in fixed order.
#include "gemv_common.cuh"

namespace dl {

constexpr int kGemvThreads = 512;
constexpr int kGemvWarps = kGemvThreads / 32;
constexpr int kGemvUnroll = 8;

template <int PRO, int EPI, int NB>
__global__ void __launch_bounds__(kGemvThreads, 1) gemvQ40Kernel(GemvArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nblk = a.n / 32;
    const uint32_t nseg = (nblk + 31) / 32;

    // ---- tile of rows owned by this CTA (pair aligned) ----
    const uint32_t nPairs = a.d / 2;
    const uint32_t pairBegin = (uint32_t)(((uint64_t)blockIdx.x * nPairs) / gridDim.x);
    const uint32_t pairEnd = (uint32_t)(((uint64_t)(blockIdx.x + 1) * nPairs) / gridDim.x);
    const uint32_t rowBase = pairBegin * 2;
    const uint32_t tileRows = (pairEnd - pairBegin) * 2;
    const uint32_t nSteps = tileRows * nseg;

    // ---- shared memory carve-up ----
    uint4 *planeA = reinterpret_cast<uint4 *>(smem);                  // [NB][nblk]
    uint4 *planeB = planeA + (size_t)NB * nblk;                       // [NB][nblk]
    float *dxs = reinterpret_cast<float *>(planeB + (size_t)NB * nblk);   // [NB][nblk]
    float *dx8 = dxs + (size_t)NB * nblk;                             // [NB][nblk]  (= 8 * dx * sum(q))
    float *partial = dx8 + (size_t)NB * nblk;                         // [maxTileRows*nseg][NB]
    float *red = partial + (size_t)a.maxTileRows * nseg * NB;         // [16]

    pdlLaunchDependents();

    uint4 q[kGemvUnroll];
    uint16_t sc[kGemvUnroll];
    auto loadGroup = [&](uint32_t s0) {
#pragma unroll
        for (int u = 0; u < kGemvUnroll; u++) {
            const uint32_t s = s0 + u * kGemvWarps;
            q[u] = make_uint4(0, 0, 0, 0);
            sc[u] = 0;
            if (s < nSteps) {
                const uint32_t r = s / nseg, seg = s - r * nseg;
                const uint32_t blk = seg * 32 + lane;
                if (blk < nblk) {
                    const uint64_t off = (uint64_t)(rowBase + r) * nblk + blk;
                    q[u] = ldgStream16(a.qs + off * 4);
                    sc[u] = ldgStreamU16(a.scales + off);
                }
            }
        }
    };

    loadGroup(warp);
    pdlWait();

    // ---- prologue: (rmsnorm) + q80 quantisation of the activation vector(s) into shared memory ----
    {
        const uint32_t nVec = a.n / 4;
#pragma unroll 1
        for (int t = 0; t < NB; t++) {
            const float4 *x4 = reinterpret_cast<const float4 *>(a.in + (size_t)t * a.inStride);
            float inv = 1.f;
            if (PRO == PRO_RMSNORM_) {
                float ss = 0.f;
                for (uint32_t i = tid; i < nVec; i += kGemvThreads) {
                    const float4 v = x4[i];
                    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
                }
                ss = blockSum512(ss, red);
                inv = rsqrtf(ss / (float)a.n + a.eps);
            }
            uint8_t *pa = reinterpret_cast<uint8_t *>(planeA + (size_t)t * nblk);
            uint8_t *pb = reinterpret_cast<uint8_t *>(planeB + (size_t)t * nblk);
            // nVec is a multiple of 8: the 8 lanes of one quant block are active together; the trip count is
            // block-uniform so full-mask shuffles are legal, out-of-range lanes just carry zeros.
            for (uint32_t base = 0; base < nVec; base += kGemvThreads) {
                const uint32_t i = base + tid;
                const bool act = i < nVec;
                float4 v = act ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                if (PRO == PRO_RMSNORM_ && act) v = rmsScale(v, reinterpret_cast<const float4 *>(a.normW)[i], inv);
                q80Pack(v, i, act, pa, pb, dxs + (size_t)t * nblk, dx8 + (size_t)t * nblk);
            }
        }
    }
    __syncthreads();

    // ---- main loop: U warp-steps per group ----
    for (uint32_t s0 = warp;;) {
#pragma unroll
        for (int u = 0; u < kGemvUnroll; u++) {
            const uint32_t s = s0 + u * kGemvWarps;
            if (s < nSteps) {   // warp-uniform
                const uint32_t r = s / nseg, seg = s - r * nseg;
                const uint32_t blk = seg * 32 + lane;
                float acc[NB];
#pragma unroll
                for (int t = 0; t < NB; t++) acc[t] = 0.f;
                if (blk < nblk) {
                    const float dw = __half2float(__ushort_as_half(sc[u]));
#pragma unroll
                    for (int t = 0; t < NB; t++) {
                        const size_t tb = (size_t)t * nblk + blk;
                        acc[t] = dw * (dxs[tb] * (float)q40q80Dot(q[u], planeA[tb], planeB[tb]) - dx8[tb]);
                    }
                }
#pragma unroll
                for (int t = 0; t < NB; t++) {
                    const float v = warpSum(acc[t]);
                    if (lane == 0) partial[(size_t)s * NB + t] = v;
                }
            }
        }
        s0 += kGemvWarps * kGemvUnroll;
        if (s0 >= nSteps) break;
        loadGroup(s0);
    }
    __syncthreads();

    // ---- epilogue: fixed-order segment sum + fused op ----
    if (EPI == EPI_SWIGLU_) {
        const uint32_t tilePairs = tileRows / 2;
        for (uint32_t i = tid; i < tilePairs * NB; i += kGemvThreads) {
            const uint32_t p = i / NB, t = i - p * NB;
            a.out[(size_t)t * a.outStride + pairBegin + p] =
                gateAct(segRowSum<NB>(partial, 2 * p, t, nseg), a.act) * segRowSum<NB>(partial, 2 * p + 1, t, nseg);
        }
    } else {
        for (uint32_t i = tid; i < tileRows * NB; i += kGemvThreads) {
            const uint32_t r = i / NB, t = i - r * NB;
            const float v = segRowSum<NB>(partial, r, t, nseg);
            float *o = a.out + (size_t)t * a.outStride + rowBase + r;
            if (EPI == EPI_RESIDUAL_) *o += v;
            else *o = v;
        }
    }
}

size_t gemvSmemBytes(uint32_t n, uint32_t maxTileRows, int nb) {
    const size_t nblk = n / 32, nseg = (nblk + 31) / 32;
    return (size_t)nb * nblk * (16 + 16 + 4 + 4) + (size_t)maxTileRows * nseg * nb * 4 + 16 * 4 + 16;
}

int launchGemvQ40Ldg(int pro, int epi, int nb, GemvArgs a, const GemvQ40Plan &p, cudaStream_t stream, bool pdl) {
    a.act = gHiddenAct;
    a.maxTileRows = p.maxTileRows;
#define DL_LAUNCH(P, E, N)                                                                                                  \
    if (pro == P && epi == E && nb == N) {                                                                                  \
        DL_CUDA_CHECK((raiseSmemLimit<gemvQ40Kernel<P, E, N>>(p.smemBytes)));                                               \
        DL_CUDA_CHECK((launchPdl(gemvQ40Kernel<P, E, N>, dim3(p.grid), dim3(kGemvThreads), p.smemBytes, stream, pdl, a)));  \
        return 0;                                                                                                           \
    }
    DL_GEMV_Q40_LDG_INSTANCES(DL_LAUNCH)
#undef DL_LAUNCH
    return -3;
}

}  // namespace dl

// Standalone entry points (tests / microbenchmarks). Engine code calls dl::gemvQ40Run directly.
// impl: 0 = auto, 1 = per-thread loads, 2 = TMA ring (returns 1 when the shape does not fit it). act: gate activation of
// EPI_SWIGLU (0 = SiLU, 1 = GELU).
DL_EXPORT int dl_gemv_q40(int pro, int epi, int nb, const void *qs, const void *scales, uint32_t d, uint32_t n,
                          const float *in, uint32_t inStride, const float *normW, float eps, float *out,
                          uint32_t outStride, int numSms, cudaStream_t stream, int pdl, int impl, uint32_t act) {
    const dl::HiddenActScope scope(act);
    dl::GemvArgs a{};
    a.qs = (const uint32_t *)qs;
    a.scales = (const __half *)scales;
    a.d = d; a.n = n;
    a.in = in; a.normW = normW; a.eps = eps;
    a.out = out; a.inStride = inStride; a.outStride = outStride;
    return dl::gemvQ40Run(pro, epi, nb, a, numSms, stream, pdl != 0, impl);
}

// The plan dl_gemv_q40 follows for a one-rank launch (launches and allocates nothing). out[8]: rc, kernel, grid, maxTileRows,
// stageRows, nStages, shared-memory bytes, launches the batch is split into.
DL_EXPORT int dl_gemv_q40_plan(int pro, int epi, int nb, uint32_t d, uint32_t n, int numSms, int impl, int *out) {
    const dl::GemvQ40Plan p = dl::planGemvQ40(pro, epi, nb, d, n, numSms, impl, true);
    const int v[8] = {p.rc, p.kernel, (int)p.grid, (int)p.maxTileRows, (int)p.stageRows, (int)p.nStages, (int)p.smemBytes, (int)p.launches};
    for (int i = 0; i < 8; i++) out[i] = v[i];
    return p.rc;
}

// One-rank fused logits + greedy token (RMSNORM prologue, EPI_ARGMAX epilogue of the TMA kernel, one token): logits into out,
// the lowest-index maximum among global rows rowOffsetGlobal + r < vocabLimit (0: no limit) into tokenOut[0], pos[0] += 1 and
// history[pos] = token while pos < historyCap. argVal / argIdx hold one entry per CTA (numSms suffice); argCounter starts at 0
// and is left at 0. Returns 1 when the shape does not fit the TMA kernel.
DL_EXPORT int dl_gemv_q40_argmax(const void *qs, const void *scales, uint32_t d, uint32_t n, const float *in, const float *normW, float eps,
                                 float *out, float *argVal, int *argIdx, unsigned int *argCounter, int *tokenOut, int *pos, int *history,
                                 uint32_t historyCap, uint32_t rowOffsetGlobal, uint32_t vocabLimit, int numSms, cudaStream_t stream) {
    dl::GemvArgs a{};
    a.qs = (const uint32_t *)qs;
    a.scales = (const __half *)scales;
    a.d = d; a.n = n;
    a.in = in; a.inStride = n; a.normW = normW; a.eps = eps;
    a.out = out; a.outStride = d;
    a.argVal = argVal; a.argIdx = argIdx; a.argCounter = argCounter;
    a.tokenOut = tokenOut; a.posInOut = pos; a.history = history; a.historyCap = historyCap;
    a.rowOffsetGlobal = rowOffsetGlobal; a.vocabLimit = vocabLimit;
    return dl::gemvQ40Tma(dl::PRO_RMSNORM_, dl::EPI_ARGMAX_, 1, a, numSms, stream, false);
}

// Logits of nb (2, 4 or 8) activation rows [nb][n] with the per-row fused arg-max (tests): out [nb][d]; row b's lowest-index maximum
// among ids < vocabLimit (0: no limit) into tokenOut[b]. argVal / argIdx hold nb x grid candidates, argCounter is zeroed and
// self-resetting. 1: the shape does not fit the TMA kernel at this width.
DL_EXPORT int dl_gemv_q40_argmax_rows(const void *qs, const void *scales, uint32_t d, uint32_t n, const float *in, const float *normW, float eps,
                                      float *out, float *argVal, int *argIdx, unsigned int *argCounter, int *tokenOut, uint32_t vocabLimit,
                                      int nb, int numSms, cudaStream_t stream) {
    if (nb != 2 && nb != 4 && nb != 8) return -4;
    dl::GemvArgs a{};
    a.qs = (const uint32_t *)qs;
    a.scales = (const __half *)scales;
    a.d = d; a.n = n;
    a.in = in; a.inStride = n; a.normW = normW; a.eps = eps;
    a.out = out; a.outStride = d;
    a.argVal = argVal; a.argIdx = argIdx; a.argCounter = argCounter; a.tokenOut = tokenOut; a.vocabLimit = vocabLimit;
    return dl::gemvQ40Tma(dl::PRO_RMSNORM_, dl::EPI_ARGMAX_ROWS_, nb, a, numSms, stream, false);
}
