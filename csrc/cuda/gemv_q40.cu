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
#include "kernels.h"

namespace dl {

enum { PRO_RMSNORM = 0, PRO_PLAIN = 1 };
enum { EPI_STORE = 0, EPI_RESIDUAL = 1, EPI_SWIGLU = 2 };

constexpr int kGemvThreads = 512;
constexpr int kGemvWarps = kGemvThreads / 32;
constexpr int kGemvUnroll = 8;

__device__ __forceinline__ float blockSum512(float v, float *red) {
    v = warpSum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < kGemvWarps) ? red[lane] : 0.f;
    t = warpSum(t);
    __syncthreads();
    return t;
}

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

    const uint32_t *qsBase = a.qs;
    const __half *scBase = a.scales;
    // Expert-indexed weights need the router output -> no prefetch before the dependency wait.
    const bool moe = a.expertIdx != nullptr;

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
                    q[u] = ldgStream16(qsBase + off * 4);
                    sc[u] = ldgStreamU16(scBase + off);
                }
            }
        }
    };

    if (!moe) loadGroup(warp);
    pdlWait();
    if (moe) {
        // one expert per launch slot; NB == 1 on this path
        const int e = a.expertIdx[a.slot];
        qsBase += (uint64_t)e * a.expertQsStride;
        scBase += (uint64_t)e * a.expertScaleStride;
        loadGroup(warp);
    }

    // ---- prologue: (rmsnorm) + q80 quantisation of the activation vector(s) into shared memory ----
    {
        const uint32_t nVec = a.n / 4;
#pragma unroll 1
        for (int t = 0; t < NB; t++) {
            const float4 *x4 = reinterpret_cast<const float4 *>(a.in + (size_t)t * a.inStride);
            float inv = 1.f;
            if (PRO == PRO_RMSNORM) {
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
                if (PRO == PRO_RMSNORM && act) {
                    const float4 w = reinterpret_cast<const float4 *>(a.normW)[i];
                    v.x = w.x * (v.x * inv); v.y = w.y * (v.y * inv); v.z = w.z * (v.z * inv); v.w = w.w * (v.w * inv);
                }
                float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
                const float d = amax / 127.f;
                const float id = d != 0.f ? 1.f / d : 0.f;
                const int q0 = __float2int_rn(v.x * id), q1 = __float2int_rn(v.y * id);
                const int q2 = __float2int_rn(v.z * id), q3 = __float2int_rn(v.w * id);
                int qsum = q0 + q1 + q2 + q3;
                qsum += __shfl_xor_sync(0xffffffffu, qsum, 1);
                qsum += __shfl_xor_sync(0xffffffffu, qsum, 2);
                qsum += __shfl_xor_sync(0xffffffffu, qsum, 4);
                if (act) {
                    const uint32_t b = i >> 3, sub = i & 7, k = sub >> 1, odd = sub & 1;
                    uint8_t *wa = pa + (size_t)b * 16 + k * 4 + odd;
                    uint8_t *wb = pb + (size_t)b * 16 + k * 4 + odd;
                    wa[0] = (uint8_t)(int8_t)q0; wa[2] = (uint8_t)(int8_t)q1;
                    wb[0] = (uint8_t)(int8_t)q2; wb[2] = (uint8_t)(int8_t)q3;
                    if (sub == 0) {
                        const float dq = __half2float(__float2half_rn(d));
                        dxs[(size_t)t * nblk + b] = dq;
                        dx8[(size_t)t * nblk + b] = dq * 8.f * (float)qsum;
                    }
                }
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
                    const uint32_t m = 0x0f0f0f0fu;
                    const uint32_t l0 = q[u].x & m, h0 = (q[u].x >> 4) & m;
                    const uint32_t l1 = q[u].y & m, h1 = (q[u].y >> 4) & m;
                    const uint32_t l2 = q[u].z & m, h2 = (q[u].z >> 4) & m;
                    const uint32_t l3 = q[u].w & m, h3 = (q[u].w >> 4) & m;
#pragma unroll
                    for (int t = 0; t < NB; t++) {
                        const uint4 A = planeA[(size_t)t * nblk + blk];
                        const uint4 B = planeB[(size_t)t * nblk + blk];
                        int dot = dp4a(l0, A.x, 0);
                        dot = dp4a(h0, B.x, dot);
                        dot = dp4a(l1, A.y, dot);
                        dot = dp4a(h1, B.y, dot);
                        dot = dp4a(l2, A.z, dot);
                        dot = dp4a(h2, B.z, dot);
                        dot = dp4a(l3, A.w, dot);
                        dot = dp4a(h3, B.w, dot);
                        acc[t] = dw * (dxs[(size_t)t * nblk + blk] * (float)dot - dx8[(size_t)t * nblk + blk]);
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
    if (EPI == EPI_SWIGLU) {
        const uint32_t tilePairs = tileRows / 2;
        for (uint32_t i = tid; i < tilePairs * NB; i += kGemvThreads) {
            const uint32_t p = i / NB, t = i - p * NB;
            float g = 0.f, up = 0.f;
            for (uint32_t sg = 0; sg < nseg; sg++) {
                g += partial[((size_t)(2 * p) * nseg + sg) * NB + t];
                up += partial[((size_t)(2 * p + 1) * nseg + sg) * NB + t];
            }
            a.out[(size_t)t * a.outStride + pairBegin + p] = gateAct(g, a.act) * up;
        }
    } else {
        for (uint32_t i = tid; i < tileRows * NB; i += kGemvThreads) {
            const uint32_t r = i / NB, t = i - r * NB;
            float v = 0.f;
            for (uint32_t sg = 0; sg < nseg; sg++) v += partial[((size_t)r * nseg + sg) * NB + t];
            float *o = a.out + (size_t)t * a.outStride + rowBase + r;
            if (EPI == EPI_RESIDUAL) {
                if (a.expertWeight) v *= a.expertWeight[t * a.kActive + a.slot];
                *o += v;
            } else {
                *o = v;
            }
        }
    }
}

size_t gemvSmemBytes(uint32_t n, uint32_t maxTileRows, int nb) {
    const size_t nblk = n / 32, nseg = (nblk + 31) / 32;
    return (size_t)nb * nblk * (16 + 16 + 4 + 4) + (size_t)maxTileRows * nseg * nb * 4 + 16 * 4 + 16;
}

template <int PRO, int EPI, int NB>
static int launchGemv(const GemvArgs &a, int grid, size_t smemBytes, cudaStream_t stream, bool pdl) {
    auto kernel = gemvQ40Kernel<PRO, EPI, NB>;
    static size_t configured = 0;   // per instantiation
    if (smemBytes > configured) {
        DL_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
        configured = smemBytes;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kGemvThreads);
    cfg.dynamicSmemBytes = smemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, a));
    return 0;
}

int launchGemvQ40Ldg(int pro, int epi, int nb, GemvArgs a, const GemvQ40Plan &p, cudaStream_t stream, bool pdl) {
    a.act = gHiddenAct;
    a.maxTileRows = p.maxTileRows;
    const int grid = (int)p.grid;
    const size_t smemBytes = p.smemBytes;
#define DL_GEMV_CASE(P, E, N) \
    if (pro == P && epi == E && nb == N) return launchGemv<P, E, N>(a, grid, smemBytes, stream, pdl);
#define DL_GEMV_NB(P, E) DL_GEMV_CASE(P, E, 1) DL_GEMV_CASE(P, E, 2) DL_GEMV_CASE(P, E, 4) DL_GEMV_CASE(P, E, 8)
    DL_GEMV_NB(PRO_RMSNORM, EPI_STORE)
    DL_GEMV_NB(PRO_PLAIN, EPI_RESIDUAL)
    DL_GEMV_NB(PRO_RMSNORM, EPI_SWIGLU)
    DL_GEMV_NB(PRO_PLAIN, EPI_STORE)
    DL_GEMV_CASE(PRO_PLAIN, EPI_SWIGLU, 1)
#undef DL_GEMV_NB
#undef DL_GEMV_CASE
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
    return dl::gemvQ40Tma(dl::PRO_RMSNORM, dl::EPI_ARGMAX_, 1, a, numSms, stream, false);
}
