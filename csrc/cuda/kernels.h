// Internal C++ interface between the kernel translation units and the engine.
#pragma once
#include "common.cuh"

namespace dl {

enum { PRO_RMSNORM_ = 0, PRO_PLAIN_ = 1 };
enum { EPI_STORE_ = 0, EPI_RESIDUAL_ = 1, EPI_SWIGLU_ = 2, EPI_ARGMAX_ = 3, EPI_MOE_DOWN_ = 4, EPI_ARGMAX_ROWS_ = 5 };
// EPI_ARGMAX: one row, the token is fed back (position advance, history); EPI_ARGMAX_ROWS: 2-8 rows, each row's arg-max to tokenOut[row]

// In-kernel one-shot all-reduce over NVLink peer memory (see the EPI_RESIDUAL epilogue of gemv_q40_tma.cu).
constexpr int kMaxRanks = 8;
// Rows of a KV-cache page of the paged slot layout (engine.cu: dl_engine_set_slot_cache).
constexpr uint32_t kPageRows = 64;
// Physical row of logical row `row` through a slot's page table.
__device__ __forceinline__ uint32_t pagedRow(const int32_t *table, uint32_t row) {
    return (uint32_t)__ldg(table + row / kPageRows) * kPageRows + row % kPageRows;
}
extern uint32_t gHiddenAct;   // process-wide gate activation (0 = SiLU, 1 = GELU), set by dl_engine_create from the model header

// Sets gHiddenAct for the launches of one stand-alone entry point and restores the engine's value afterwards (the launchers read
// it on the host when they fill the kernel arguments).
struct HiddenActScope {
    uint32_t saved;
    explicit HiddenActScope(uint32_t act) : saved(gHiddenAct) { gHiddenAct = act; }
    ~HiddenActScope() { gHiddenAct = saved; }
};

struct ArArgs {
    uint32_t nRanks, rank, parity, maxCtas;
    uint32_t slotStride;          // words per (parity, source rank) slot = maxBatch * dim
    uint32_t dim;                 // words between tokens inside a slot
    uint64_t *slots[kMaxRanks];   // rank r's LL slot area, mapped into this process: [2][nRanks][slotStride] x (f32 payload, flag)
    uint64_t *cand[kMaxRanks];    // rank r's arg-max candidates: [nRanks] x (f32 value, index + 1)
    uint64_t *slotsMc;            // NVLS multicast mapping of the slot area (one multimem.st reaches every rank), or null
};

struct GemvArgs {
    const uint32_t *qs;
    const __half *scales;
    uint32_t d, n;
    const float *in;
    const float *normW;
    float eps;
    float *out;
    uint32_t inStride, outStride;
    uint32_t maxTileRows;
    const int *expertIdx;
    uint32_t kActive;
    uint64_t expertQsStride, expertScaleStride;
    const float *expertWeight;
    // EPI_ARGMAX (TMA kernel, nb == 1): logits are stored and the greedy token is selected in the same launch
    float *argVal;            // [grid] per-CTA best value
    int *argIdx;              // [grid] per-CTA best index
    unsigned int *argCounter; // zero-initialised, self-resetting
    int *tokenOut, *posInOut, *history;
    uint32_t historyCap;
    uint32_t rowOffsetGlobal; // added to row indices (vocab slice offset under tensor parallelism)
    uint64_t *trace;          // optional 4-slot timeline record for this launch
    // Mixture-of-experts launches (moeCtasPerSlot > 0, nb == 1): CTA b works for routing slot b / moeCtasPerSlot on the row
    // tile b % moeCtasPerSlot of expert expertIdx[slot]; experts outside [moeFirstExpert, +moeNumLocal) are skipped (EP).
    uint32_t moeCtasPerSlot, moeFirstExpert, moeNumLocal;
    uint32_t inSlotStride, outSlotStride;   // floats between slots of the input (w2) / output (w13) buffers
    float *moeScratch;          // [kActive][d] weighted per-slot products (EPI_MOE_DOWN)
    unsigned int *moeCounters;  // [moeCtasPerSlot], zero-initialised, self-resetting
    ArArgs ar;                // ar.nRanks > 1: EPI_RESIDUAL sums the partial products of all ranks before the residual add
    uint32_t act;             // gate activation of EPI_SWIGLU (filled in by the launchers from gHiddenAct)
    uint32_t vocabLimit;      // EPI_ARGMAX: rows (global index) >= vocabLimit never win (model vocabulary padded beyond the tokenizer's); 0 = no limit
};
// What a q40 GEMV launch runs (planGemvQ40, gemv_q40_tma.cu). impl: 0 = TMA ring if the shape fits it, else per-thread loads;
// 1 = per-thread loads only; 2 = TMA ring only (rc 1: the shape does not fit it).
// When no kernel fits nb tokens in shared memory and `split` is set, the batch runs as `launches` consecutive launches of
// nb / launches tokens each; the other fields describe one such launch. rc < 0: the launch is refused.
struct GemvQ40Plan {
    int rc, kernel;                 // kernel: 1 = per-thread loads (gemvQ40Kernel), 2 = TMA ring (gemvQ40TmaKernel)
    uint32_t grid, maxTileRows;
    uint32_t stageRows, nStages;    // TMA ring geometry (0 for kernel 1)
    uint32_t smemBytes, launches;
};
// moeCtasPerSlot / kActive: mixture-of-experts launches (TMA only, nb == 1): row tiles per routing slot and slots.
GemvQ40Plan planGemvQ40(int pro, int epi, int nb, uint32_t d, uint32_t n, int numSms, int impl, bool split,
                        uint32_t moeCtasPerSlot = 0, uint32_t kActive = 0);
size_t gemvSmemBytes(uint32_t n, uint32_t maxTileRows, int nb);   // per-thread-load kernel
int launchGemvQ40Ldg(int pro, int epi, int nb, GemvArgs a, const GemvQ40Plan &p, cudaStream_t stream, bool pdl);
int launchGemvQ40Tma(int pro, int epi, int nb, GemvArgs a, const GemvQ40Plan &p, cudaStream_t stream, bool pdl);
// Plans and launches. A batch is split only on one rank (ar.nRanks <= 1), outside expert launches and for the STORE, RESIDUAL and
// SWIGLU epilogues, whose tokens are independent; the in-kernel all-reduce indexes its slots per token.
int gemvQ40Run(int pro, int epi, int nb, const GemvArgs &a, int numSms, cudaStream_t stream, bool pdl, int impl);
inline int gemvQ40Tma(int pro, int epi, int nb, const GemvArgs &a, int numSms, cudaStream_t stream, bool pdl) {    // 1: shape unsupported
    return gemvQ40Run(pro, epi, nb, a, numSms, stream, pdl, 2);
}

// f32 / f16 weight files (gemv_dense.cu): wtype 1 = f32, 2 = f16; a.qs is the row-major [d][n] matrix
int gemvDense(int wtype, int pro, int epi, int nb, GemvArgs a, int numSms, cudaStream_t stream, bool pdl);
size_t gemvDenseSmemBytes(uint32_t n, uint32_t maxTileRows, int nb);

// ---- KV-cache storage --------------------------------------------------------------------------------------------------------------
// Every cache below is head-major [nKvHeads][seqLen][headDim]. Its rows are bf16 (kScale / vScale null), or q80 (EngineConfig::kvType
// 1): int8 values in the value plane (kCache / vCache) and one f16 scale per 32 values in a separate scale plane
// [nKvHeads][seqLen][headDim / 32], so value rows stay 16-byte aligned for bulk copies. A row is rounded once, where it is written,
// with the GEMV q80 prologue's arithmetic: d = amax / 127, q = rint(x / d), scale f16(d); readers see q * f16(d).
// Element offsets apply to both planes: value element e has its scale at e / 32.

// Rounds the DPL consecutive values a lane holds of one row (a 32-value block spans 32 / DPL neighbouring lanes) to q80 in place:
// v becomes q * f16(d). All 32 lanes of the warp take part.
template <int DPL>
__device__ __forceinline__ void q80RoundLane(float (&v)[DPL], int8_t (&q)[DPL], __half &d16) {
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < DPL; i++) amax = fmaxf(amax, fabsf(v[i]));
#pragma unroll
    for (int o = 1; o < 32 / DPL; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = amax / 127.f;
    const float id = d != 0.f ? 1.f / d : 0.f;
    d16 = __float2half_rn(d);
    const float dq = __half2float(d16);
#pragma unroll
    for (int i = 0; i < DPL; i++) {
        const int qi = __float2int_rn(v[i] * id);
        q[i] = (int8_t)qi;
        v[i] = (float)qi * dq;
    }
}

// int8 value i (0..3) of the packed word w as f32, exactly. An int-to-float conversion (I2F) runs at a fraction of the FP32 rate
// on sm_90, and the decode kernels convert every cached value once per q-head: instead the biased byte (x + 128) goes into the
// low mantissa byte of 2^23 (one PRMT) and one FADD removes 2^23 + 128.
__device__ __forceinline__ float q8ToFloat(uint32_t w, int i) {
    return __uint_as_float(__byte_perm(w ^ 0x80808080u, 0x4B000000u, 0x7650u | (uint32_t)i)) - 8388736.f;
}

// The DPL values of one cache row at element offset e (DPL in {2, 4}, e a multiple of DPL) as f32.
template <int DPL, bool Q8>
__device__ __forceinline__ void loadKv(const void *plane, const __half *scale, size_t e, float (&o)[DPL]) {
    if constexpr (Q8) {
        const float d = __half2float(scale[e / 32]);
        const int8_t *p = reinterpret_cast<const int8_t *>(plane) + e;
        const uint32_t w = DPL == 4 ? *reinterpret_cast<const uint32_t *>(p) : (uint32_t)*reinterpret_cast<const uint16_t *>(p);
#pragma unroll
        for (int i = 0; i < DPL; i++) o[i] = q8ToFloat(w, i) * d;
    } else {
        const __nv_bfloat16 *p = reinterpret_cast<const __nv_bfloat16 *>(plane) + e;
        if constexpr (DPL == 4) {
            const uint2 r = *reinterpret_cast<const uint2 *>(p);
            const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.x));
            const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.y));
            o[0] = a0.x; o[1] = a0.y; o[2] = a1.x; o[3] = a1.y;
        } else {
            const uint32_t r = *reinterpret_cast<const uint32_t *>(p);
            const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r));
            o[0] = a0.x; o[1] = a0.y;
        }
    }
}

// Rounds the DPL values a lane holds of a new row to the cache's storage in place (all 32 lanes take part) and, if `store`, writes
// them at element offset e. For bf16 every lane rounds its own values; for q80 the lane that holds the start of a block writes its scale.
template <int DPL, bool Q8>
__device__ __forceinline__ void roundStoreKv(float (&v)[DPL], void *plane, __half *scale, size_t e, bool store) {
    if constexpr (Q8) {
        int8_t q[DPL];
        __half d16;
        q80RoundLane<DPL>(v, q, d16);
        if (store) {
            int8_t *p = reinterpret_cast<int8_t *>(plane) + e;
            if constexpr (DPL == 4) *reinterpret_cast<char4 *>(p) = make_char4(q[0], q[1], q[2], q[3]);
            else *reinterpret_cast<char2 *>(p) = make_char2(q[0], q[1]);
            if (e % 32 == 0) scale[e / 32] = d16;
        }
    } else {
        __nv_bfloat162 b[DPL / 2];
#pragma unroll
        for (int k = 0; k < DPL / 2; k++) {
            b[k] = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
            const float2 f = __bfloat1622float2(b[k]);
            v[2 * k] = f.x; v[2 * k + 1] = f.y;
        }
        if (store) {
            __nv_bfloat162 *p = reinterpret_cast<__nv_bfloat162 *>(reinterpret_cast<__nv_bfloat16 *>(plane) + e);
#pragma unroll
            for (int k = 0; k < DPL / 2; k++) p[k] = b[k];
        }
    }
}

struct RopeKvArgs {
    float *qkv;
    uint32_t qkvStride;
    const int *pos;
    const float *rope;
    const float *qNorm;
    const float *kNorm;
    float eps;
    uint32_t nHeads, nKvHeads, headDim, seqLen;
    void *kCache, *vCache;       // bf16, or the int8 value planes of a q80 cache
    __half *kScale, *vScale;     // q80 scale planes; null: bf16 cache
    // Choice steps (several sequences at one rotary position): token t stores its K/V row at pos[t] + t * rowStride, and tokens
    // whose bit is set in inactiveMask store nothing. Both 0 for a plain batch of consecutive tokens.
    uint32_t rowStride, inactiveMask;
    // Slots steps (attn_decode.cu): token t stores its K/V row pos[t] at element offset t * slotStride (slot t, seqLen = the slot's
    // length L). 0 for every other caller.
    uint64_t slotStride;
};
int launchRopeKv(const RopeKvArgs &a, int nb, cudaStream_t stream, bool pdl);
// Paged slots (slotStride 0, seqLen = the rows of the whole layer plane): token t stores its logical row pos[t] at physical row
// pageTable[t * pageTableStride + pos / 64] * 64 + pos % 64 (stride 0: every token through one slot's table). The paged kernels take
// these derived structs so that the others keep their argument layout, and with it their code.
struct PagedRopeKvArgs : RopeKvArgs {
    const int32_t *pageTable;
    uint32_t pageTableStride;
};
int launchRopeKvPaged(const PagedRopeKvArgs &a, int nb, cudaStream_t stream, bool pdl);

// Attention of B choices that share the prompt rows [0, P] of the cache (attn_decode.cu). Query row b (choice b, rotary position
// P + 1 + j, already normalised and rotated by ropeKvKernel) attends to [0, P] and to its own rows [P + 1 + b * C, P + 1 + b * C + j].
// A CTA owns (KV head, prefix split) and serves all B * nHeads / nKvHeads query rows of that head, so each prefix row is read
// once per step. The last split also runs the per-choice suffixes; the last CTA to finish merges the splits.
struct ChoiceAttnArgs {
    const float *qkv;
    uint32_t qkvStride;
    const void *kCache, *vCache;
    const __half *kScale, *vScale;   // q80 scale planes; null: bf16 cache
    uint32_t nHeads, nKvHeads, headDim, seqLen, nSplits;
    uint32_t B, P, C, j;
    uint32_t inactiveMask;   // rows whose bit is set skip their suffix; their output is not meaningful
    float *partial;          // >= B * nHeads * nSplits * (headDim + 2) floats
    unsigned int *counters;  // [nKvHeads], zero-initialised, self-resetting
    float *out;              // [B][outStride], head h at columns h * headDim
    uint32_t outStride;
};
int launchChoiceAttn(const ChoiceAttnArgs &a, cudaStream_t stream, bool pdl);

// Attention of B independent sequences, row b in KV-cache slot b (attn_decode.cu): slot b is the [nKvHeads][L][headDim] block at element
// offset b * slotStride of the cache; query row b (position pos[b], already normalised and rotated by ropeKvKernel) attends to rows
// [0, pos[b]] of its slot. A CTA owns (KV head, split, row) and serves the nHeads / nKvHeads q-heads of that KV head.
struct SlotAttnArgs {
    const float *qkv;
    uint32_t qkvStride;
    const int *pos;          // [B]
    const void *kCache, *vCache;
    const __half *kScale, *vScale;   // q80 scale planes; null: bf16 cache
    uint64_t slotStride;     // elements between slots: nKvHeads * L * headDim
    uint32_t nHeads, nKvHeads, headDim, L, nSplits;
    uint32_t B, inactiveMask;   // rows whose bit is set do nothing; their output is not meaningful
    float *partial;          // >= B * nHeads * nSplits * (headDim + 2) floats
    unsigned int *counters;  // [B][nKvHeads], zero-initialised, self-resetting
    float *out;              // [B][outStride], head h at columns h * headDim
    uint32_t outStride;
};
int launchSlotAttn(const SlotAttnArgs &a, cudaStream_t stream, bool pdl);
// Paged slots (slotStride unused): every layer plane holds planeRows rows per KV head, and row b's logical row r lives at physical
// row pageTable[b * pageStride + r / 64] * 64 + r % 64. L is the longest a slot may grow.
struct PagedSlotAttnArgs : SlotAttnArgs {
    const int32_t *pageTable;
    uint32_t pageStride, planeRows;
};
int launchSlotAttnPaged(const PagedSlotAttnArgs &a, cudaStream_t stream, bool pdl);

struct AttnArgs {
    const float *qkv;
    uint32_t qkvStride;
    const int *pos;
    const void *kCache, *vCache;
    const __half *kScale, *vScale;   // q80 scale planes; null: bf16 cache
    uint32_t nHeads, nKvHeads, headDim, seqLen, nSplits;
    float *partial;
    unsigned int *counters;
    float *out;
    uint32_t outStride;
    __nv_bfloat16 *outBf16;   // if set, the result is written here (bf16) instead of `out`
};
int launchAttnDecode(const AttnArgs &a, int nb, cudaStream_t stream, bool pdl);

// Prompt-chunk attention on the tensor cores (attn_prefill_tc.cu, wgmma): T consecutive tokens at positions p0.., causal, GQA heads packed on MMA-M.
struct AttnPrefillArgs {
    const float *qkv;            // [T][qkvStride] f32, q rows already normalised + rotated; K/V of the chunk already in the cache
    uint32_t qkvStride;
    uint32_t T, p0;
    uint32_t nHeads, nKvHeads, headDim, seqLen;
    const void *kCache, *vCache;            // [nKvHeads][seqLen][headDim]
    const __half *kScale, *vScale;          // q80 scale planes; null: bf16 cache
    __nv_bfloat16 *out;          // [T][outStride], head h at columns h * headDim
    uint32_t outStride;
    // Paged slot (set): seqLen is the rows of the whole layer plane, and logical row r lives at physical row
    // pageTable[r / 64] * 64 + r % 64; pages up to row p0 + T - 1 must be mapped.
    const int32_t *pageTable;
};
int launchAttnPrefillTc(const AttnPrefillArgs &a, cudaStream_t stream, bool pdl = false);   // 1: shape not covered

// Single-token decode attention with QK-norm + RoPE + KV-cache append fused in (no separate rope kernel).
struct AttnFusedArgs {
    const float *qkv;        // raw q|k|v row of the token (f32, straight from the QKV GEMV)
    const int *pos;
    const float *rope;       // [seqLen][hd/2][2]
    const float *qNorm, *kNorm;
    float eps;
    void *kCache, *vCache;
    __half *kScale, *vScale;   // q80 scale planes; null: bf16 cache
    uint32_t nHeads, nKvHeads, headDim, seqLen, nSplits;
    float *partial;
    unsigned int *counters;
    float *out;
    uint64_t *trace;
};
int launchAttnFused(const AttnFusedArgs &a, cudaStream_t stream, bool pdl);

struct RouterArgs {
    const float *x;            // [nb][dim] residual stream
    const float *normW;        // [dim]
    const float *gate;         // [nExperts][dim] f32
    float eps;
    uint32_t dim, nExperts, k;
    float *logits;             // [nb][nExperts] scratch
    unsigned int *counter;     // [nb], zero-initialised, self-resetting
    int *expertIdx;            // [nb][k]
    float *expertWeight;       // [nb][k]
};
int launchMoeRouter(const RouterArgs &a, int nb, cudaStream_t stream, bool pdl);

// Token embedding table (f32 [vocab][dim]). Tensor parallel: sharded by vocabulary rows over the ranks' peer-mapped memory — rank r
// holds rows [r * rowsPerRank, (r + 1) * rowsPerRank) and every rank reads the row of the current token straight from its owner over
// NVLink (reference K1: the root embeds and broadcasts x, src/llm.cpp:248-256; here a 16 KB peer load replaces 2.1 GB x N of replicas).
struct EmbTable {
    const float *shard[kMaxRanks];   // shard[0] is the whole table when rowsPerRank == 0
    uint32_t rowsPerRank;
    __host__ __device__ const float *row(uint32_t tok, uint32_t dim) const {
        if (rowsPerRank == 0) return shard[0] + (size_t)tok * dim;
        const uint32_t r = tok / rowsPerRank;
        return shard[r] + (size_t)(tok - r * rowsPerRank) * dim;
    }
};
int launchEmbedding(const EmbTable &table, const int *tokens, float *x, uint32_t dim, uint32_t xStride, uint32_t vocab, int nb,
                    cudaStream_t stream);
int launchArgmaxAdvance(const float *logits, uint32_t vocab, int *tokenOut, int *pos, int *history, uint32_t historyCap,
                        cudaStream_t stream, bool pdl);   // single rank only: the index is local to `logits`
int launchArgmaxRows(const float *logits, uint32_t stride, uint32_t vocab, int nb, int *out, cudaStream_t stream, bool pdl);

// Speculative decoding (speculative.cu). Result block of a round, int32: [0] accepted drafts a, [1] emitted tokens a + 1, [2] drafts k,
// [3] position of the last emitted token, [kSpecResultHead + i] emitted token i.
constexpr uint32_t kSpecMaxDraft = 7, kSpecResultHead = 4, kSpecResultWords = kSpecResultHead + kSpecMaxDraft + 1;
struct SpecAcceptArgs {
    const int *verifyTokens;            // [k + 1] the target's arg-max after rows t, d1..dk
    int *targetTokens, *targetPos;      // [k + 1]: t, d1..dk and p (row 0); next round: tokens[0], pos[0]
    int *targetHistory;                 // history[q] = the token at position q (may be null)
    uint32_t historyCap;
    int *draftTokens, *draftPos, *draftHistory;
    uint32_t draftHistoryCap;
    uint32_t k;                         // 1 .. kSpecMaxDraft
    int *result;                        // [kSpecResultWords]
};
int launchSpecStage(const SpecAcceptArgs &a, cudaStream_t stream);
int launchSpecAccept(const SpecAcceptArgs &a, cudaStream_t stream);

// Device-side temperature / top-p sampler and the logits gather that feeds it under tensor parallelism (sampler.cu)
// Optional per-request controls, applied to every logit before temperature (float32, round to nearest, no contraction):
//   x = l[t] + bias[t] (bias non-null); if c[t] > 0: x = x - c[t] * frequency, then x = x - presence.
// counts row b (counts + b * countsStride) holds how often row b has drawn each token; every draw increments it. With controls
// the temperature may be 0: the token is then the arg-max of the transformed logits (lowest index among ties).
struct SampleControls {
    const float *bias;        // [n] or null
    uint32_t *counts;         // [rows][countsStride] or null
    uint32_t countsStride;
    float presence, frequency;
    uint32_t biasStride;      // row b's bias at bias + b * biasStride (0: one bias for every row)
};
// The controls' transform of logit i; explicit roundings because the library is built with --use_fast_math. `drawn`: an id whose
// count holds one draw to leave out (the log-probabilities read a row's counts after its draw incremented them), -1: none.
__device__ __forceinline__ float controlled(const SampleControls &c, float x, uint32_t i, int drawn = -1) {
    if (c.bias) x = __fadd_rn(x, c.bias[i]);
    if (c.counts) {
        uint32_t k = c.counts[i];
        if ((int)i == drawn && k > 0) k--;
        if (k > 0) x = __fsub_rn(__fsub_rn(x, __fmul_rn((float)k, c.frequency)), c.presence);
    }
    return x;
}
// Optional sampling filters of a temperature > 0 draw. With e[i] = exp(x[i] / T - max(x / T)) (the sampler's unnormalised
// probabilities), the candidate set S keeps the ids that pass both active filters: top_k keeps the topK first ids in the order
// (e desc, id asc), min_p keeps e[i] >= f32(minP * max e). Ids outside S get e = 0 before the normaliser; a nucleus draw then
// drops below (1 - top-p) / (|S| - 1), and |S| == 1 returns that id. topK 0 (or >= n) and minP 0 are off: the draw is exactly
// the unfiltered one. minP must lie in [0, 1]. Temperature 0 ignores the filters (the arg-max is always in S).
struct SampleFilters {
    uint32_t topK;
    float minP;
};
bool sampleFiltersValid(const SampleFilters &f);   // minP in [0, 1]
int launchSample(const float *logits, float *probs, uint32_t n, float temperature, float topp, unsigned long long *rng, int *tokenOut, int *pos,
                 int *history, uint32_t historyCap, const unsigned int *gatherFlag, unsigned int *gatherEpoch, uint32_t nRanks,
                 cudaStream_t stream, const SampleControls *controls = nullptr, const SampleFilters *filters = nullptr);
int launchLogitsGather(const float *local, uint32_t v0, uint32_t rank, uint32_t nRanks, float *gatherMc, float *const *gatherUcDev,
                       unsigned int *flagMc, unsigned int *const *flagUcDev, unsigned int *blockCounter, cudaStream_t stream, uint32_t rows = 1);
// B draws, one CTA per row: row b reads logits + b * logitsStride (0: every row draws from the same logits), uses rng[b] and writes
// tokenOut[b]. Rows whose bit is set in inactiveMask draw nothing and keep their generator state. No position advance.
// rowParams (device [B][4], may be null): row b's {temperature, top-p, presence, frequency} in place of the scalar arguments and the
// controls' penalties; a row with temperature 0 draws the arg-max (lowest index among ties).
// filters (host, may be null): the filters of every row. rowFilters (device [B], may be null): row b's filters in their place.
int launchSampleRows(const float *logits, uint32_t logitsStride, float *probs, uint32_t n, float temperature, float topp, unsigned long long *rng,
                     int *tokenOut, uint32_t B, uint32_t inactiveMask, const unsigned int *gatherFlag, unsigned int *gatherEpoch, uint32_t nRanks,
                     cudaStream_t stream, const SampleControls *controls = nullptr, const float *rowParams = nullptr,
                     const SampleFilters *filters = nullptr, const SampleFilters *rowFilters = nullptr);

// Per-token log-probabilities (logprobs.cu): logprob(i) = x[i] - logsumexp(x[0..n)) of the row that drew token chosen[b], where x
// is the logits row after the controls (the values the sampler draws from, before temperature). One CTA per row b < B whose bit
// is set in rowMask; other rows read nothing. Row b reads logits + b * logitsStride (0: every row reads one row), its controls as
// launchSampleRows does (rowParams: per-row penalties at [b][2..3]) with its counts read after the draw, and writes kLogprobsWords
// int32 words at out + b * kLogprobsWords: {chosen id, its logprob (f32 bits), k, 0, then k (id, logprob bits) pairs}: the k[b]
// largest logprobs in the order (value desc, id asc). The chosen token's logprob is bitwise its value in that list.
constexpr int kLogprobsMaxTop = 20;
constexpr int kLogprobsWords = 4 + 2 * kLogprobsMaxTop;
int launchLogprobsRows(const float *logits, uint32_t logitsStride, uint32_t n, uint32_t B, uint32_t rowMask, const int *k, const int *chosen,
                       int32_t *out, cudaStream_t stream, const SampleControls *controls = nullptr, const float *rowParams = nullptr);

// Persistent decode kernel (mega_decode.cu)
struct MegaLayer {
    const uint8_t *qkvQs, *qkvSc, *woQs, *woSc, *w13Qs, *w13Sc, *w2Qs, *w2Sc;
    const float *norm0, *norm1, *qNorm, *kNorm;
    void *kCache, *vCache;     // bf16, or the int8 value planes of a q80 cache (MegaArgs::kvScales)
};

struct MegaKvScales {          // q80 caches: the scale planes of one layer
    __half *k, *v;
};

struct MegaPhase {   // host-computed geometry of one GEMV phase (QKV, WO, W1|W3, W2, logits)
    uint32_t d, n, nblk, nseg;
    uint32_t stageRows;            // rows per ring fill (multiple of 4)
    uint32_t pairsQ, pairsRem;     // row pairs per CTA: CTA b owns pairsQ + (b < pairsRem) pairs starting at b*pairsQ + min(b, pairsRem)
    uint32_t recipNseg, gInc, segInc, rotInc;   // step -> (row group, segment) bookkeeping without divisions
};

struct MegaArgs {
    const MegaLayer *layers;     // [nLayers] in global memory
    uint32_t nLayers, dim, nHeads, nKvHeads, headDim, ffDim, vocab, vocabFull, seqLen, nSplits;
    float eps;
    EmbTable embedding;
    const float *finalNorm, *rope;
    const uint8_t *wclsQs, *wclsSc;
    int *tokens, *pos, *history;
    float *logits;
    uint2 *xW2;                  // second residual buffer (barrier-free hand-off experiment, flags bit 0)
    uint32_t flags;
    uint2 *xW, *qkvW, *zW;       // phase-crossing vectors as LL words {f32, epoch} (engine-owned, see mega_decode.cu)
    float *hF;                   // SwiGLU vector: plain f32 behind a fenced barrier (too large to pay the 2x LL footprint)
    unsigned int *launchSeq;     // device-resident launch counter (epoch base)
    unsigned int *abortFlag;     // host-mapped: set by a wait loop that ran out of its spin budget
    unsigned long long *syncNs;  // device accumulator: ns CTA 0 spent waiting for peer ranks in the all-reduce epilogues (null: off)
    float *attnPartial;
    unsigned int *attnCounters;
    float *argVal;
    int *argIdx;
    unsigned int *argCounter;
    unsigned int *gridCounter;   // zeroed by a memset node before every launch
    uint32_t stageBytes, nStages, planeBlocks, partialFloats;   // shared-memory geometry (host computed)
    uint32_t maxInflight;        // producer pacing: bulk-copy fills outstanding per CTA (0 = the whole ring)
    MegaPhase ph[5];
    uint32_t rowOffsetGlobal;
    uint32_t greedyAdvance;      // 1: publish the arg-max token and advance the position on the device
    uint32_t act, vocabLimit;    // see GemvArgs
    uint64_t *trace;
    uint32_t traceCtas, traceStride;   // CTAs 0..traceCtas-1 record their phase stamps at trace[cta * traceStride + slot]
    uint32_t traceProdSlot;      // != 0: first producer slot of a CTA's trace row (megaTraceProdSlot; all-CTA tracing only)
    ArArgs ar;
    const MegaKvScales *kvScales;   // [nLayers] in global memory: the caches are q80; null: bf16
};

// Trace row of one CTA of the persistent kernel: 18 * nLayers + 5 consumer phase stamps, then (from this slot on, 8-aligned) two
// producer counters per weight phase k = 4 * layer + {QKV, WO, W1|W3, W2}, k = 4 * nLayers for the logits: at 2k the ns the
// producer waited for a free ring stage, at 2k + 1 the ns it waited on the in-flight cap. A layer's K/V fills count towards its QKV phase.
inline uint32_t megaTraceProdSlot(uint32_t nLayers) { return (18 * nLayers + 5 + 7) / 8 * 8; }
inline uint32_t megaTraceRowSlots(uint32_t nLayers) { return megaTraceProdSlot(nLayers) + 2 * (4 * nLayers + 1); }

int launchMegaDecode(MegaArgs m, int numSms, cudaStream_t stream);

// tensor-core prefill GEMM (gemm_q40_tc.cu, wgmma)
enum { GEPI_STORE_F32_ = 0, GEPI_RESIDUAL_ = 1, GEPI_SWIGLU_BF16_ = 2 };
int gemmQ40Tc(int epi, const void *qs, const void *scales, uint32_t d, uint32_t n, const void *act, uint32_t actStride, uint32_t T,
              void *out, uint32_t outStride, int numSms, cudaStream_t stream, bool pdl);
int gemmQ40TcGrouped(int epi, const void *qs, const void *scales, uint32_t nGroups, uint32_t grpRows, uint32_t n, const void *act,
                     uint32_t actStride, uint32_t rowsTotal, uint32_t maxTokens, const int *grpCount, const int *grpOffset, void *out,
                     uint32_t outStride, int numSms, cudaStream_t stream);   // 1: shape not covered
// Mixture-of-experts feed-forward over a prompt chunk (moe_prefill.cu)
struct MoePrefillArgs {
    float *x;                     // [T][dim] residual stream, updated in place
    void *xnScratch;              // bf16 [T][dim]
    const float *norm, *gate;     // ffn rms-norm weight [dim], router gate [nExperts][dim] f32
    const void *w13Qs, *w13Sc, *w2Qs, *w2Sc;
    uint32_t T, dim, ff, nExperts, k, firstLocal, nLocal;
    float eps;
    int numSms;
    ArArgs ar;                    // nRanks > 1: partial sums are all-reduced over peer memory inside the combine kernel
};
int moePrefillFfn(const MoePrefillArgs &a, cudaStream_t stream);   // 1: shape not covered
// Test read-back of the last moePrefillFfn call's routing and per-pair SwiGLU output (see moe_prefill.cu); -1: scratch too small
int moePrefillScratchRead(uint32_t T, uint32_t k, uint32_t nExperts, uint32_t ff, float *logits, int *ids, float *weights,
                          __nv_bfloat16 *hPairs, cudaStream_t stream);
// Launch with the programmatic-dependent-launch attribute: the kernel may start while its predecessor in the stream is still running
// and must execute griddepcontrol.wait (pdlWait) before touching anything the predecessor produces or still reads.
template <typename... KArgs, typename... Args>
inline cudaError_t launchPdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
// Raises Kernel's dynamic shared-memory limit to `bytes` when a launch needs more than any earlier one (one record per kernel).
template <auto Kernel>
inline cudaError_t raiseSmemLimit(size_t bytes) {
    static size_t configured = 0;
    if (bytes <= configured) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) configured = bytes;
    return e;
}

int launchArResidual(float *x, const float *partial, uint32_t dim, uint32_t T, const ArArgs &ar, cudaStream_t stream, bool pdl = false);   // x += all-reduce(partial)
int launchRmsNormBf16(const float *x, uint32_t xStride, const float *w, void *y, uint32_t yStride, uint32_t n, float eps, uint32_t T,
                      cudaStream_t stream, bool pdl = false);

}  // namespace dl
