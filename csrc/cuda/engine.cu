// Per-rank inference engine: owns the kernel schedule of one forward pass, its scratch, arena layout, prompt chunking and decode graph.
//
// Role in the reference: NnExecutor + NnCpuDevice/NnVulkanDevice + the `start/att/ff/end` segments emitted by
// buildLlmNet (src/nn/nn-executor.cpp:45-207, src/llm.cpp:247-603) — ~26 barrier-separated ops per layer driven
// by an interpreter. Here a forward pass is a fixed sequence of 5 fused kernels per layer, chained with
// programmatic dependent launch, and the single-token step is captured once into a CUDA graph whose inputs
// (token id, position) live in device memory so the graph replays without host round trips:
// the sampling kernel writes the next token and advances the position on the device.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "engine_api.h"
#include "kernels.h"

namespace dl {

uint32_t gHiddenAct = 0;

static_assert(kApiMaxRanks == kMaxRanks, "engine_api.h and kernels.h disagree on the rank limit");
static_assert(kApiLogprobsWords == kLogprobsWords && kApiLogprobsMaxTop == kLogprobsMaxTop, "engine_api.h and kernels.h disagree on logprobs");

// The client's GlobalPtrs and the scratch buffers the engine allocates for itself (allocScratch).
struct Buffers : GlobalPtrs {
    float *qkv, *z, *h;          // [maxBatch][qkvDim | qDim | ff] (h: at least nActiveExperts rows)
    float *attnPartial;          // [maxBatch][nHeads][nSplits][hd+2]
    unsigned int *attnCounters;  // [maxBatch][nHeads]
    // MoE scratch
    int *expertIdx;              // [maxBatch][nActive]
    float *expertWeight;         // [maxBatch][nActive]
    float *routerLogits;         // [maxBatch][nExperts]
    unsigned int *routerCounter; // [maxBatch]
    float *moeScratch;           // [nActive][dim]
    unsigned int *moeCounters;   // [256]
    // prefill (tensor-core GEMM path) buffers, maxPrefill tokens
    int *pTokens, *pPos;         // [maxPrefill]
    float *px, *pqkv;            // [maxPrefill][dim | max(qkvDim, dim)] f32
    void *pxn, *pzb, *phb;       // bf16 [maxPrefill][dim | qDim | ff]
    float *pAttnPartial;         // [maxPrefill][nHeads][hd+2]
    unsigned int *pAttnCounters; // [maxPrefill][nHeads]
    // fused arg-max scratch
    float *argVal;               // [256 >= numSms]
    int *argIdx;                 // [256]
    unsigned int *argCounter;    // [4]
};

// The client's CommPtrs and the arena layout the engine derives from its configuration (arenaLayout).
struct Comm : CommPtrs {
    uint32_t maxCtas, slotStride, prefillSlotStride;
    uint64_t slotsOff, flagsOff, candValOff, gatherOff, prefillSlotsOff;
};

struct Engine {
    EngineConfig cfg{};
    Comm comm{};
    std::vector<LayerPtrs> layers;
    Buffers g{};
    uint8_t *scratch = nullptr;    // the allocation behind the Buffers scratch pointers
    uint32_t prefillMinTc = 9;     // shortest prompt chunk on the tensor cores (0: never)
    cudaGraphExec_t decodeGraph = nullptr;
    cudaStream_t captureStream = nullptr;
    int lastError = 0;
    uint64_t *trace = nullptr;   // device buffer [maxLaunches][4] of globaltimer stamps (optional)
    uint32_t traceCap = 0;
    bool traceAllCtas = false;   // persistent kernel: every CTA records its phase stamps (skew analysis, tools/trace_mega.py --all)
    MegaLayer *megaLayers = nullptr;   // device copy of the per-layer pointer table for the persistent decode kernel
    MegaKvScales *megaKvScales = nullptr;   // q80 caches: device copy of the per-layer scale planes (null: bf16)
    unsigned int *megaCounter = nullptr;
    uint2 *megaX2 = nullptr;
    uint32_t megaFlags = 0;            // DL_MEGA_FLAGS (bit 0: barrier-free LL hand-off)
    uint2 *megaX = nullptr, *megaQkv = nullptr, *megaZ = nullptr, *megaH = nullptr;   // LL vectors of the persistent kernel
    unsigned int *megaSeq = nullptr;
    unsigned int *abortHost = nullptr, *abortDev = nullptr;   // mapped pinned word: device wait loops report a blown spin budget here
    uint32_t megaInflight = 1;         // DL_MEGA_INFLIGHT: producer pacing of the persistent kernel (0 = unpaced; DESIGN.md §7)
    uint32_t megaCtas = 0;             // DL_MEGA_CTAS: grid size override of the persistent kernel (0 = one CTA per SM)
    bool useMega = false;
    bool lastDecodeMega = false, megaFallbackWarned = false;   // did the last single-token forward run on the persistent kernel?
    // device sampler state (sampler.cu)
    unsigned long long *rngState = nullptr;
    float *probScratch = nullptr;
    unsigned int *gatherEpoch = nullptr, *gatherBlockCounter = nullptr;
    float **gatherUcDev = nullptr;
    unsigned int **flagUcDev = nullptr;
    uint32_t vocabLimit = 0;     // 0 = none; otherwise the greedy arg-max ignores vocabulary rows >= vocabLimit
    // sampling controls (dl_engine_set_sampling_controls), allocated on first use: count rows [1 + kChoiceRngSlots][vocabFull]
    // (row 0: single sequence, row 1 + b: choice b) and a dense bias [vocabFull]
    uint32_t *ctlCounts = nullptr;
    float *ctlBias = nullptr;
    bool ctlActive = false, ctlBiasActive = false;
    float ctlPresence = 0.f, ctlFrequency = 0.f;
    dl::SampleFilters filters{};       // top_k / min_p of the single sequence and the choices (dl_engine_set_sampling_filters)
    // KV-cache slots (dl_engine_set_slots): slots > 1 splits every layer's cache into `slots` blocks of slotLen rows
    uint32_t slots = 1, slotLen = 0;
    float *slotParams = nullptr;       // [kChoiceRngSlots][4] per-slot {temperature, top-p, presence, frequency}
    float *slotBias = nullptr;         // [kChoiceRngSlots][vocabFull] per-slot logit bias
    dl::SampleFilters *slotFiltersDev = nullptr;   // [kChoiceRngSlots] per-slot top_k / min_p (dl_engine_slot_filters)
    dl::SampleFilters slotFilters[8] = {};         // host copy: the step reads the device array only while one is on
    int32_t *slotStage = nullptr;      // pinned [3][kChoiceRngSlots]: tokens, positions in; drawn tokens out
    cudaEvent_t slotStaged = nullptr;  // the uploads of the staged tokens / positions are done: the buffer may be rewritten
    int slotLogprobs[8] = {-1, -1, -1, -1, -1, -1, -1, -1};   // per-slot top_logprobs k (-1: no logprobs), one per slot
    int32_t *slotLpDev = nullptr, *slotLpHost = nullptr;   // [kChoiceRngSlots][kLogprobsWords] results of a slots step (device, pinned)
    // Paged slots (dl_engine_set_slot_cache): every layer plane is a pool of nPages 64-row pages shared by the slots; slot s maps its
    // logical page i to physical page pageHost[s * nPages + i] (i < slotPages[s]; -1 past them). The device copy is refreshed on the
    // stream of the next call that reads it (uploadPages).
    bool pagedSlots = false;
    uint32_t nPages = 0;
    int32_t *pageDev = nullptr, *pageHost = nullptr;   // [kChoiceRngSlots][nPages] (device, pinned)
    std::vector<uint32_t> slotPages;
    std::vector<uint8_t> pageUsed;
    bool pagesDirty = false;
    cudaEvent_t pagesStaged = nullptr;   // the last upload has read pageHost
    bool tcAttn = true;          // prefill attention on the tensor cores (DL_NO_TC_ATTN=1: per-token CUDA-core kernel)
    bool fusedAttn = true;       // debugging switch (DL_NO_FUSED_ATTN)
    uint64_t serial = 0;         // unique per engine of the process (a round graph names its draft by it)
    uint32_t graphGen = 0;       // bumped whenever captured launches of this engine go stale (dropGraph)
    struct Spec *spec = nullptr; // speculative rounds with this engine as the target (dl_spec_round), allocated on first use
};

// The target's state of speculative rounds: per-row arg-max scratch of the verify GEMV, its tokens, the accept kernel's result
// block, a pinned staging block and one round graph per draft length.
struct Spec {
    uint8_t *dev = nullptr;            // one allocation: argVal [8][256], argIdx [8][256], counter, verify tokens [8], result block
    float *argVal = nullptr;
    int *argIdx = nullptr;
    unsigned int *argCounter = nullptr;
    int *verifyTok = nullptr, *result = nullptr;
    int32_t *stage = nullptr;          // pinned: [0] token, [1] position in; [kSpecResultHead..] the result block out
    cudaGraphExec_t graph[kSpecMaxDraft + 1] = {};
    uint64_t graphDraft[kSpecMaxDraft + 1] = {};          // serial of the draft engine the graph was captured with
    uint32_t graphGen[kSpecMaxDraft + 1][2] = {};         // graphGen of the target and the draft at capture
};

#define DL_TRY(expr)                    \
    do {                                \
        const int _r = (expr);          \
        if (_r != 0) return _r;         \
    } while (0)

static EmbTable embTable(const Engine &e) {
    EmbTable t{};
    t.rowsPerRank = e.g.embRowsPerRank;
    if (t.rowsPerRank == 0) t.shard[0] = e.g.embedding;
    else for (int r = 0; r < kMaxRanks; r++) t.shard[r] = e.g.embeddingPeers[r];
    return t;
}

static void fillAr(const Engine &e, ArArgs &ar, uint32_t parity) {
    const Comm &c = e.comm;
    ar.nRanks = c.nRanks; ar.rank = c.rank; ar.parity = parity; ar.maxCtas = c.maxCtas; ar.slotStride = c.slotStride; ar.dim = e.cfg.dim;
    ar.slotsMc = c.mcArena ? (uint64_t *)((uint8_t *)c.mcArena + c.slotsOff) : nullptr;
    for (uint32_t r = 0; r < c.nRanks && r < (uint32_t)kMaxRanks; r++) {
        uint8_t *base = (uint8_t *)c.arena[r];
        ar.slots[r] = (uint64_t *)(base + c.slotsOff);
        ar.cand[r] = (uint64_t *)(base + c.candValOff);
    }
}

static uint32_t localVocabLimit(const Engine &e) {
    return (e.vocabLimit && e.vocabLimit < e.cfg.vocab) ? e.vocabLimit : e.cfg.vocab;
}

static int gemvSel(const Engine &e, int pro, int epi, int nb, const GemvArgs &a, int numSms, cudaStream_t stream, bool pdl) {
    if (e.cfg.wType != 0) return gemvDense((int)e.cfg.wType, pro, epi, nb, a, numSms, stream, pdl);
    if (a.ar.nRanks > 1) {   // the in-kernel all-reduce lives in the TMA kernel only
        const int r = gemvQ40Tma(pro, epi, nb, a, numSms, stream, pdl);
        return r == 1 ? -30 : r;
    }
    return gemvQ40Run(pro, epi, nb, a, numSms, stream, pdl, 0);
}

// Mixture-of-experts feed-forward of one token, all buffers explicit (the engine's and those of tests/test_gpu_moe.py).
struct MoeDecodeArgs {
    const float *x;                       // [dim] residual stream (router and W1|W3 input)
    float *out;                           // [dim] the weighted expert sum is added here
    const float *norm, *gate;             // ffn rms-norm weight [dim], router gate [nExperts][dim] f32
    const void *w13Qs, *w13Sc, *w2Qs, *w2Sc;   // [nLocal][2*ff][dim] gate/up interleaved, [nLocal][dim][ff]
    int wType;                            // 0 = q40 device layout; 1 = f32, 2 = f16 dense rows (the *Sc pointers are unused)
    uint32_t dim, ff, nExperts, k, firstLocal, nLocal;
    float eps;
    float *routerLogits;                  // [nExperts]
    unsigned int *routerCounter;          // [1], zero-initialised, self-resetting
    int *expertIdx;                       // [k]
    float *expertWeight;                  // [k]
    float *h;                             // [k][ff] SwiGLU output per routing slot
    float *moeScratch;                    // [k][dim] weighted per-slot products
    unsigned int *moeCounters;            // [numSms / k], zero-initialised, self-resetting
    uint32_t numSms;                      // CTAs per routing slot = numSms / k (at least 1)
    uint64_t *trace13, *trace2;
    ArArgs ar;                            // nRanks > 1: all-reduce in the W2 epilogue
};

// router -> k x (W1|W3 -> silu*up) -> k x W2; the weighted expert sum is *added* to `out`. q40 experts run on the TMA GEMV,
// f32 / f16 experts on the expert-routed mode of the dense GEMV (gemv_dense.cu).
static int moeDecodeFfn(const MoeDecodeArgs &m, cudaStream_t stream, bool pdl) {
    RouterArgs ro{};
    ro.x = m.x; ro.normW = m.norm; ro.gate = m.gate; ro.eps = m.eps; ro.dim = m.dim; ro.nExperts = m.nExperts;
    ro.k = m.k; ro.logits = m.routerLogits; ro.counter = m.routerCounter; ro.expertIdx = m.expertIdx; ro.expertWeight = m.expertWeight;
    DL_TRY(launchMoeRouter(ro, 1, stream, pdl));
    const uint32_t perSlot = m.numSms / m.k > 0 ? m.numSms / m.k : 1;
    GemvArgs a{};
    a.qs = (const uint32_t *)m.w13Qs; a.scales = (const __half *)m.w13Sc; a.d = 2 * m.ff; a.n = m.dim;
    a.in = m.x; a.inStride = m.dim; a.normW = m.norm; a.eps = m.eps; a.out = m.h; a.outStride = m.ff; a.trace = m.trace13;
    a.moeCtasPerSlot = perSlot; a.kActive = m.k; a.expertIdx = m.expertIdx; a.outSlotStride = m.ff;
    a.expertQsStride = (uint64_t)2 * m.ff * (m.dim / 8); a.expertScaleStride = (uint64_t)2 * m.ff * (m.dim / 32);
    a.moeFirstExpert = m.firstLocal; a.moeNumLocal = m.nLocal;
    if (m.wType != 0) DL_TRY(gemvDense(m.wType, PRO_RMSNORM_, EPI_SWIGLU_, 1, a, (int)m.numSms, stream, pdl));
    else { const int r = gemvQ40Tma(PRO_RMSNORM_, EPI_SWIGLU_, 1, a, (int)m.numSms, stream, pdl); if (r != 0) return r == 1 ? -31 : r; }
    a = GemvArgs{};
    a.qs = (const uint32_t *)m.w2Qs; a.scales = (const __half *)m.w2Sc; a.d = m.dim; a.n = m.ff;
    a.in = m.h; a.inStride = m.ff; a.inSlotStride = m.ff; a.out = m.out; a.outStride = m.dim; a.trace = m.trace2;
    a.moeCtasPerSlot = perSlot; a.kActive = m.k; a.expertIdx = m.expertIdx; a.expertWeight = m.expertWeight;
    a.expertQsStride = (uint64_t)m.dim * (m.ff / 8); a.expertScaleStride = (uint64_t)m.dim * (m.ff / 32);
    a.moeFirstExpert = m.firstLocal; a.moeNumLocal = m.nLocal; a.moeScratch = m.moeScratch; a.moeCounters = m.moeCounters;
    a.ar = m.ar;
    if (m.wType != 0) DL_TRY(gemvDense(m.wType, PRO_PLAIN_, EPI_MOE_DOWN_, 1, a, (int)m.numSms, stream, pdl));
    else { const int r = gemvQ40Tma(PRO_PLAIN_, EPI_MOE_DOWN_, 1, a, (int)m.numSms, stream, pdl); if (r != 0) return r == 1 ? -32 : r; }
    return 0;
}

// Mixture-of-experts feed-forward of the engine's token: the weighted expert sum is *added* to `out` (the residual stream, or a
// zeroed partial buffer on the NCCL path), all-reduced in the epilogue if asked.
static int runMoe(Engine &e, const LayerPtrs &L, float *out, bool fusedAr, uint64_t *trace13, uint64_t *trace2, cudaStream_t stream,
                  bool pdl) {
    const EngineConfig &c = e.cfg;
    MoeDecodeArgs m{};
    m.x = e.g.x; m.out = out; m.norm = L.norm1; m.gate = L.moeGate;
    m.w13Qs = L.w13Qs; m.w13Sc = L.w13Sc; m.w2Qs = L.w2Qs; m.w2Sc = L.w2Sc; m.wType = (int)c.wType;
    m.dim = c.dim; m.ff = c.ffDim; m.nExperts = c.nExperts; m.k = c.nActiveExperts; m.firstLocal = c.moeFirstExpert; m.nLocal = c.moeNumLocal;
    m.eps = c.eps; m.routerLogits = e.g.routerLogits; m.routerCounter = e.g.routerCounter; m.expertIdx = e.g.expertIdx;
    m.expertWeight = e.g.expertWeight; m.h = e.g.h; m.moeScratch = e.g.moeScratch; m.moeCounters = e.g.moeCounters; m.numSms = c.numSms;
    m.trace13 = trace13; m.trace2 = trace2;
    if (fusedAr) fillAr(e, m.ar, 1);
    return moeDecodeFfn(m, stream, pdl);
}

// One token through the persistent kernel (dense models, nb == 1). Returns 1 when the shape is not supported.
static int engineDecodeMega(Engine &e, bool greedyAdvance, cudaStream_t stream) {
    const EngineConfig &c = e.cfg;
    if (!e.megaLayers || c.nExperts > 0 || c.wType != 0) return 1;
    MegaArgs m{};
    m.layers = e.megaLayers; m.nLayers = c.nLayers; m.dim = c.dim; m.nHeads = c.nHeads; m.nKvHeads = c.nKvHeads; m.headDim = c.headDim;
    m.ffDim = c.ffDim; m.vocab = c.vocab; m.vocabFull = e.g.vocabFull; m.seqLen = c.seqLen; m.nSplits = c.nSplits; m.eps = c.eps;
    m.embedding = embTable(e); m.finalNorm = e.g.finalNorm; m.rope = e.g.rope;
    m.wclsQs = (const uint8_t *)e.g.wclsQs; m.wclsSc = (const uint8_t *)e.g.wclsSc;
    m.tokens = e.g.tokens; m.pos = e.g.pos; m.history = e.g.history;
    m.logits = e.g.logits; m.maxInflight = e.megaInflight;
    m.xW = e.megaX; m.xW2 = e.megaX2; m.flags = e.megaFlags; m.qkvW = e.megaQkv; m.zW = e.megaZ; m.hF = (float *)e.megaH; m.launchSeq = e.megaSeq; m.abortFlag = e.abortDev;
    m.syncNs = (e.comm.nRanks > 1 && e.megaSeq) ? (unsigned long long *)(e.megaSeq + 2) : nullptr;
    m.attnPartial = e.g.attnPartial; m.attnCounters = e.g.attnCounters;
    m.argVal = e.g.argVal; m.argIdx = e.g.argIdx; m.argCounter = e.g.argCounter; m.gridCounter = e.megaCounter;
    m.rowOffsetGlobal = c.rank * c.vocab; m.greedyAdvance = greedyAdvance ? 1u : 0u; m.vocabLimit = e.vocabLimit;
    m.trace = e.trace;
    m.kvScales = e.megaKvScales;
    m.traceCtas = e.traceAllCtas ? c.numSms : 1u;
    m.traceStride = e.traceAllCtas ? (uint32_t)(((size_t)e.traceCap * 4) / c.numSms) : 0u;
    m.traceProdSlot = (e.trace && m.traceStride >= megaTraceRowSlots(c.nLayers)) ? megaTraceProdSlot(c.nLayers) : 0u;
    if (e.comm.nRanks > 1) fillAr(e, m.ar, 0);
    return launchMegaDecode(m, (int)(e.megaCtas ? e.megaCtas : c.numSms), stream);
}

// Geometry of a choices step (see attn_decode.cu): nb rows at rotary position P + 1 + j, row b stored at P + 1 + b * C + j.
struct ChoiceStep { uint32_t P, C, j, inactiveMask; };

// A slots step (see attn_decode.cu): row b is KV-cache slot b at position pos[b].
struct SlotStep { uint32_t inactiveMask; };

static uint64_t slotElems(const Engine &e) { return (uint64_t)e.cfg.nKvHeads * e.slotLen * e.cfg.headDim; }

// The layer's K/V caches from element cacheOff on, in the engine's storage (bf16, or q80 value and scale planes).
struct KvPtrs { void *k, *v; __half *ks, *vs; };
static KvPtrs layerKv(const Engine &e, const LayerPtrs &L, uint64_t cacheOff) {
    if (e.cfg.kvType == 0) return {(__nv_bfloat16 *)L.kCache + cacheOff, (__nv_bfloat16 *)L.vCache + cacheOff, nullptr, nullptr};
    return {(int8_t *)L.kCache + cacheOff, (int8_t *)L.vCache + cacheOff, (__half *)L.kScale + cacheOff / 32, (__half *)L.vScale + cacheOff / 32};
}

// QK-norm + RoPE + K/V write of layer L over the q|k|v rows `qkv` at positions `pos`, into the cache that starts cacheOff elements
// into the layer's K/V and holds seqLen rows per KV head. rowStride, slotStride and inactiveMask are left 0 for the caller to set.
static RopeKvArgs layerRopeKv(const Engine &e, const LayerPtrs &L, float *qkv, const int *pos, uint64_t cacheOff, uint32_t seqLen) {
    const EngineConfig &c = e.cfg;
    RopeKvArgs r{};
    r.qkv = qkv; r.qkvStride = (c.nHeads + 2 * c.nKvHeads) * c.headDim; r.pos = pos; r.rope = e.g.rope; r.qNorm = L.qNorm; r.kNorm = L.kNorm;
    r.eps = c.eps; r.nHeads = c.nHeads; r.nKvHeads = c.nKvHeads; r.headDim = c.headDim; r.seqLen = seqLen;
    const KvPtrs kv = layerKv(e, L, cacheOff);
    r.kCache = kv.k; r.vCache = kv.v; r.kScale = kv.ks; r.vScale = kv.vs;
    return r;
}

// logitsMode: 0 = none (prefill chunk), 1 = logits of the last token in the batch into logits[0], 2 = all tokens, 3 = all tokens
// and the arg-max of every row into spec->verifyTok (the verify step of a speculative round: nb >= 2, one rank, dense q40).
// ch: a choices step instead of a batch of consecutive tokens (logitsMode 2, dense layers only); sl: a slots step (same limits).
static int engineForward(Engine &e, int nb, int logitsMode, bool greedyAdvance, cudaStream_t stream, const ChoiceStep *ch = nullptr,
                         const SlotStep *sl = nullptr) {
    const EngineConfig &c = e.cfg;
    const bool pdl = c.usePdl != 0;
    const uint32_t qDim = c.nHeads * c.headDim, kvDim = c.nKvHeads * c.headDim, qkvDim = qDim + 2 * kvDim;
    if (nb < 1 || (uint32_t)nb > c.maxBatch || (nb & (nb - 1))) return -10;
    e.lastDecodeMega = false;
    if ((ch || sl) && (c.nExperts > 0 || logitsMode != 2 || greedyAdvance)) return -14;
    if (logitsMode == 3 && (nb < 2 || !e.spec || greedyAdvance || c.wType != 0 || c.nExperts > 0 || e.comm.nRanks > 1)) return -73;
    if (nb == 1 && logitsMode == 1 && e.useMega) {
        const int r = engineDecodeMega(e, greedyAdvance, stream);
        if (r != 1) { e.lastDecodeMega = r == 0; return r; }
        if (!e.megaFallbackWarned) {
            std::fprintf(stderr, "dl_engine: the persistent decode kernel cannot run this configuration (shape, shared memory or co-residency); "
                                 "using the multi-kernel path\n");
            e.megaFallbackWarned = true;
        }
    }
    uint32_t slot = 0;
    auto nextTrace = [&]() -> uint64_t * { uint64_t *t = (e.trace && slot < e.traceCap) ? e.trace + (size_t)slot * 4 : nullptr; slot++; return t; };

    DL_TRY(launchEmbedding(embTable(e), e.g.tokens, e.g.x, c.dim, c.dim, e.g.vocabFull, nb, stream));
    for (uint32_t l = 0; l < c.nLayers; l++) {
        const LayerPtrs &L = e.layers[l];
        GemvArgs a{};
        // 1. rmsnorm -> q80 -> QKV
        a.qs = (const uint32_t *)L.qkvQs; a.scales = (const __half *)L.qkvSc; a.d = qkvDim; a.n = c.dim;
        a.in = e.g.x; a.inStride = c.dim; a.normW = L.norm0; a.eps = c.eps; a.out = e.g.qkv; a.outStride = qkvDim; a.trace = nextTrace();
        DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_STORE_, nb, a, c.numSms, stream, pdl));
        if (sl) {
            // 2+3. qk-norm + rope + K/V append at row pos[b] of slot b, then attention of each row over its own slot
            RopeKvArgs r = layerRopeKv(e, L, e.g.qkv, e.g.pos, 0, e.pagedSlots ? c.seqLen : e.slotLen);
            if (!e.pagedSlots) r.slotStride = slotElems(e);
            r.inactiveMask = sl->inactiveMask;
            SlotAttnArgs t{};
            t.qkv = e.g.qkv; t.qkvStride = qkvDim; t.pos = e.g.pos; t.kCache = r.kCache; t.vCache = r.vCache; t.kScale = r.kScale; t.vScale = r.vScale; t.slotStride = r.slotStride;
            t.nHeads = c.nHeads; t.nKvHeads = c.nKvHeads; t.headDim = c.headDim; t.L = e.slotLen; t.nSplits = c.nSplits;
            t.B = (uint32_t)nb; t.inactiveMask = sl->inactiveMask;
            t.partial = e.g.attnPartial; t.counters = e.g.attnCounters; t.out = e.g.z; t.outStride = qDim;
            if (e.pagedSlots) {
                PagedRopeKvArgs pr{};
                static_cast<RopeKvArgs &>(pr) = r;
                pr.pageTable = e.pageDev; pr.pageTableStride = e.nPages;
                DL_TRY(launchRopeKvPaged(pr, nb, stream, pdl));
                PagedSlotAttnArgs pt{};
                static_cast<SlotAttnArgs &>(pt) = t;
                pt.pageTable = e.pageDev; pt.pageStride = e.nPages; pt.planeRows = c.seqLen;
                DL_TRY(launchSlotAttnPaged(pt, stream, pdl));
            } else {
                DL_TRY(launchRopeKv(r, nb, stream, pdl));
                DL_TRY(launchSlotAttn(t, stream, pdl));
            }
        } else if (ch) {
            // 2+3. qk-norm + rope + K/V append at the choices' own rows, then attention over the shared prompt + own rows
            RopeKvArgs r = layerRopeKv(e, L, e.g.qkv, e.g.pos, 0, c.seqLen);
            r.rowStride = ch->C; r.inactiveMask = ch->inactiveMask;
            DL_TRY(launchRopeKv(r, nb, stream, pdl));
            ChoiceAttnArgs t{};
            t.qkv = e.g.qkv; t.qkvStride = qkvDim; t.kCache = r.kCache; t.vCache = r.vCache; t.kScale = r.kScale; t.vScale = r.vScale;
            t.nHeads = c.nHeads; t.nKvHeads = c.nKvHeads; t.headDim = c.headDim; t.seqLen = c.seqLen; t.nSplits = c.nSplits;
            t.B = (uint32_t)nb; t.P = ch->P; t.C = ch->C; t.j = ch->j; t.inactiveMask = ch->inactiveMask;
            t.partial = e.g.attnPartial; t.counters = e.g.attnCounters; t.out = e.g.z; t.outStride = qDim;
            DL_TRY(launchChoiceAttn(t, stream, pdl));
        } else if (nb == 1 && e.fusedAttn) {
            // 2+3. qk-norm + rope + kv append + attention in one launch
            AttnFusedArgs f{};
            f.qkv = e.g.qkv; f.pos = e.g.pos; f.rope = e.g.rope; f.qNorm = L.qNorm; f.kNorm = L.kNorm; f.eps = c.eps;
            const KvPtrs kv = layerKv(e, L, 0);
            f.kCache = kv.k; f.vCache = kv.v; f.kScale = kv.ks; f.vScale = kv.vs;
            f.nHeads = c.nHeads; f.nKvHeads = c.nKvHeads; f.headDim = c.headDim; f.seqLen = c.seqLen; f.nSplits = c.nSplits;
            f.partial = e.g.attnPartial; f.counters = e.g.attnCounters; f.out = e.g.z; f.trace = nextTrace();
            DL_TRY(launchAttnFused(f, stream, pdl));
        } else {
            // 2. qk-norm + rope + kv write
            const RopeKvArgs r = layerRopeKv(e, L, e.g.qkv, e.g.pos, 0, c.seqLen);
            DL_TRY(launchRopeKv(r, nb, stream, pdl));
            // 3. attention
            AttnArgs t{};
            t.qkv = e.g.qkv; t.qkvStride = qkvDim; t.pos = e.g.pos; t.kCache = r.kCache; t.vCache = r.vCache; t.kScale = r.kScale; t.vScale = r.vScale;
            t.nHeads = c.nHeads; t.nKvHeads = c.nKvHeads; t.headDim = c.headDim; t.seqLen = c.seqLen; t.nSplits = c.nSplits;
            t.partial = e.g.attnPartial; t.counters = e.g.attnCounters; t.out = e.g.z; t.outStride = qDim;
            DL_TRY(launchAttnDecode(t, nb, stream, pdl));
        }
        // 4. q80 -> WO, residual add
        a = GemvArgs{};
        a.qs = (const uint32_t *)L.woQs; a.scales = (const __half *)L.woSc; a.d = c.dim; a.n = qDim;
        a.in = e.g.z; a.inStride = qDim; a.out = e.g.x; a.outStride = c.dim; a.trace = nextTrace();
        if (e.comm.nRanks > 1) fillAr(e, a.ar, 0);
        DL_TRY(gemvSel(e, PRO_PLAIN_, EPI_RESIDUAL_, nb, a, c.numSms, stream, pdl));
        if (c.nExperts > 0) {
            // 5-7. mixture of experts: router -> k x (W1|W3 -> silu*up) -> k x W2, weighted sum, residual (+ all-reduce)
            if (nb != 1) return -13;
            nextTrace();
            uint64_t *t13 = nextTrace(), *t2 = nextTrace();
            DL_TRY(runMoe(e, L, e.g.x, e.comm.nRanks > 1, t13, t2, stream, pdl));
            continue;
        }
        // 5. rmsnorm -> q80 -> W1|W3 -> silu*up
        a = GemvArgs{};
        a.qs = (const uint32_t *)L.w13Qs; a.scales = (const __half *)L.w13Sc; a.d = 2 * c.ffDim; a.n = c.dim;
        a.in = e.g.x; a.inStride = c.dim; a.normW = L.norm1; a.eps = c.eps; a.out = e.g.h; a.outStride = c.ffDim; a.trace = nextTrace();
        DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_SWIGLU_, nb, a, c.numSms, stream, pdl));
        // 6. q80 -> W2, residual add
        a = GemvArgs{};
        a.qs = (const uint32_t *)L.w2Qs; a.scales = (const __half *)L.w2Sc; a.d = c.dim; a.n = c.ffDim;
        a.in = e.g.h; a.inStride = c.ffDim; a.out = e.g.x; a.outStride = c.dim; a.trace = nextTrace();
        if (e.comm.nRanks > 1) fillAr(e, a.ar, 1);
        DL_TRY(gemvSel(e, PRO_PLAIN_, EPI_RESIDUAL_, nb, a, c.numSms, stream, pdl));
    }
    if (logitsMode != 0) {
        GemvArgs a{};
        a.qs = (const uint32_t *)e.g.wclsQs; a.scales = (const __half *)e.g.wclsSc; a.d = c.vocab; a.n = c.dim;
        a.normW = e.g.finalNorm; a.eps = c.eps; a.inStride = c.dim; a.outStride = c.vocab; a.out = e.g.logits; a.trace = nextTrace();
        if (logitsMode == 1) {
            a.in = e.g.x + (size_t)(nb - 1) * c.dim;
            int r = 1;
            if (greedyAdvance && c.wType == 0) {
                // logits + greedy sampling + position advance in one launch
                a.argVal = e.g.argVal; a.argIdx = e.g.argIdx; a.argCounter = e.g.argCounter;
                a.tokenOut = e.g.tokens; a.posInOut = e.g.pos; a.history = e.g.history; a.historyCap = c.seqLen;
                a.rowOffsetGlobal = c.rank * c.vocab; a.vocabLimit = e.vocabLimit;
                if (e.comm.nRanks > 1) fillAr(e, a.ar, 0);
                r = gemvQ40Tma(PRO_RMSNORM_, EPI_ARGMAX_, 1, a, c.numSms, stream, pdl);
                if (r < 0) return r;
            }
            if (r == 1) {
                // the stand-alone arg-max kernel sees this rank's vocabulary slice only: under tensor parallelism the ranks would
                // pick different (local) ids, so the non-fused route is refused there instead of silently diverging
                if (greedyAdvance && e.comm.nRanks > 1) return -33;
                a.argVal = nullptr; a.argIdx = nullptr; a.argCounter = nullptr; a.tokenOut = nullptr; a.posInOut = nullptr; a.history = nullptr;
                a.ar = ArArgs{};
                DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_STORE_, 1, a, c.numSms, stream, pdl));
                if (greedyAdvance)
                    DL_TRY(launchArgmaxAdvance(e.g.logits, localVocabLimit(e), e.g.tokens, e.g.pos, e.g.history, c.seqLen, stream, pdl));
            }
        } else if (logitsMode == 3) {
            a.in = e.g.x;
            a.argVal = e.spec->argVal; a.argIdx = e.spec->argIdx; a.argCounter = e.spec->argCounter; a.tokenOut = e.spec->verifyTok;
            a.vocabLimit = e.vocabLimit;
            const int r = gemvQ40Tma(PRO_RMSNORM_, EPI_ARGMAX_ROWS_, nb, a, c.numSms, stream, pdl);
            if (r < 0) return r;
            if (r == 1) {
                // the fused per-row arg-max needs all nb rows' partial sums in one CTA's shared memory (Llama-3.3-70B, Qwen3-14B
                // logits at nb = 8 do not fit): the STORE GEMV, which may split the batch, then one arg-max CTA per row
                a.argVal = nullptr; a.argIdx = nullptr; a.argCounter = nullptr; a.tokenOut = nullptr;
                DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_STORE_, nb, a, c.numSms, stream, pdl));
                DL_TRY(launchArgmaxRows(e.g.logits, c.vocab, localVocabLimit(e), nb, e.spec->verifyTok, stream, pdl));
            }
        } else {
            a.in = e.g.x;
            DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_STORE_, nb, a, c.numSms, stream, pdl));
            if (greedyAdvance) {
                if (e.comm.nRanks > 1) return -33;
                DL_TRY(launchArgmaxAdvance(e.g.logits, localVocabLimit(e), e.g.tokens, e.g.pos, e.g.history, c.seqLen, stream, pdl));
            }
        }
    }
    return 0;
}

// Prompt chunk of T <= maxPrefill tokens on the tensor-core path. Logits (optional) are produced for the last token.
// slot >= 0: the chunk goes into KV-cache slot `slot` (a cache of its own of slotLen rows).
static int enginePrefill(Engine &e, uint32_t T, uint32_t p0, int wantLogits, cudaStream_t stream, int slot = -1) {
    const EngineConfig &c = e.cfg;
    const Buffers &g = e.g;
    const bool pdl = c.usePdl != 0;   // every kernel of this chain waits (griddepcontrol.wait) before touching its predecessor's data
    const uint32_t qDim = c.nHeads * c.headDim, kvDim = c.nKvHeads * c.headDim, qkvDim = qDim + 2 * kvDim;
    if (T < 1 || T > c.maxPrefill) return -11;
    if (c.wType != 0) return -35;   // tensor-core path: q40 matrices
    const bool paged = slot >= 0 && e.pagedSlots;
    const uint32_t seqLen = slot >= 0 && !paged ? e.slotLen : c.seqLen;   // rows a KV head's plane holds
    const uint64_t cacheOff = slot >= 0 && !paged ? (uint64_t)slot * slotElems(e) : 0;
    if (slot >= 0 && ((uint32_t)slot >= e.slots || p0 + T > (paged ? e.slotPages[slot] * kPageRows : seqLen))) return -60;
    if (paged && !e.tcAttn) return -69;
    const int32_t *pages = paged ? e.pageDev + (size_t)slot * e.nPages : nullptr;
    const bool tp = e.comm.nRanks > 1;
    ArArgs arP{};
    if (tp) {
        if (e.comm.prefillSlotStride < T * c.dim) return -12;
        fillAr(e, arP, 0);
        arP.slotStride = e.comm.prefillSlotStride;
        for (uint32_t r = 0; r < e.comm.nRanks; r++) arP.slots[r] = (uint64_t *)((uint8_t *)e.comm.arena[r] + e.comm.prefillSlotsOff);
        arP.slotsMc = e.comm.mcArena ? (uint64_t *)((uint8_t *)e.comm.mcArena + e.comm.prefillSlotsOff) : nullptr;
    }
    DL_TRY(launchEmbedding(embTable(e), g.pTokens, g.px, c.dim, c.dim, g.vocabFull, (int)T, stream));
    for (uint32_t l = 0; l < c.nLayers; l++) {
        const LayerPtrs &L = e.layers[l];
        DL_TRY(launchRmsNormBf16(g.px, c.dim, L.norm0, g.pxn, c.dim, c.dim, c.eps, T, stream, pdl));
        DL_TRY(gemmQ40Tc(GEPI_STORE_F32_, L.qkvQs, L.qkvSc, qkvDim, c.dim, g.pxn, c.dim, T, g.pqkv, qkvDim, c.numSms, stream, pdl));
        const RopeKvArgs r = layerRopeKv(e, L, g.pqkv, g.pPos, cacheOff, seqLen);
        if (paged) {
            PagedRopeKvArgs pr{};
            static_cast<RopeKvArgs &>(pr) = r;
            pr.pageTable = pages;
            DL_TRY(launchRopeKvPaged(pr, (int)T, stream, pdl));
        } else DL_TRY(launchRopeKv(r, (int)T, stream, pdl));
        int attnRc = 1;
        if (e.tcAttn) {
            // tensor-core attention over the whole chunk: the tokens of a chunk sit at consecutive positions p0 .. p0 + T - 1
            AttnPrefillArgs ap{};
            ap.qkv = g.pqkv; ap.qkvStride = qkvDim; ap.T = T; ap.p0 = p0; ap.nHeads = c.nHeads; ap.nKvHeads = c.nKvHeads;
            ap.headDim = c.headDim; ap.seqLen = seqLen; ap.kCache = r.kCache; ap.vCache = r.vCache; ap.kScale = r.kScale; ap.vScale = r.vScale;
            ap.out = (__nv_bfloat16 *)g.pzb; ap.outStride = qDim; ap.pageTable = pages;
            attnRc = launchAttnPrefillTc(ap, stream, pdl);
            if (attnRc < 0) return attnRc;
            if (attnRc == 1 && paged) return -69;
        }
        if (attnRc == 1) {
            AttnArgs t{};
            t.qkv = g.pqkv; t.qkvStride = qkvDim; t.pos = g.pPos; t.kCache = r.kCache; t.vCache = r.vCache; t.kScale = r.kScale; t.vScale = r.vScale;
            t.nHeads = c.nHeads; t.nKvHeads = c.nKvHeads; t.headDim = c.headDim; t.seqLen = seqLen; t.nSplits = 1;
            t.partial = g.pAttnPartial; t.counters = g.pAttnCounters; t.out = nullptr; t.outStride = qDim; t.outBf16 = (__nv_bfloat16 *)g.pzb;
            DL_TRY(launchAttnDecode(t, (int)T, stream, pdl));
        }
        // tensor parallel: partial product into the (now free) qkv buffer with all SMs / split-K, then all-reduce + residual over
        // peer memory as its own kernel
        if (tp) {
            arP.parity = 0;
            DL_TRY(gemmQ40Tc(GEPI_STORE_F32_, L.woQs, L.woSc, c.dim, qDim, g.pzb, qDim, T, g.pqkv, c.dim, c.numSms, stream, pdl));
            DL_TRY(launchArResidual(g.px, g.pqkv, c.dim, T, arP, stream, pdl));
        } else DL_TRY(gemmQ40Tc(GEPI_RESIDUAL_, L.woQs, L.woSc, c.dim, qDim, g.pzb, qDim, T, g.px, c.dim, c.numSms, stream, pdl));
        if (c.nExperts > 0) {
            // mixture of experts: route the whole chunk, sort the (token, expert) pairs, grouped tensor-core GEMMs, weighted combine
            MoePrefillArgs mo{};
            mo.x = g.px; mo.xnScratch = g.pxn; mo.norm = L.norm1; mo.gate = L.moeGate; mo.w13Qs = L.w13Qs; mo.w13Sc = L.w13Sc;
            mo.w2Qs = L.w2Qs; mo.w2Sc = L.w2Sc; mo.T = T; mo.dim = c.dim; mo.ff = c.ffDim; mo.nExperts = c.nExperts; mo.k = c.nActiveExperts;
            mo.firstLocal = c.moeFirstExpert; mo.nLocal = c.moeNumLocal; mo.eps = c.eps; mo.numSms = (int)c.numSms;
            if (tp) { arP.parity = 1; mo.ar = arP; }
            const int mr = moePrefillFfn(mo, stream);
            if (mr != 0) return mr == 1 ? -36 : mr;
            continue;
        }
        DL_TRY(launchRmsNormBf16(g.px, c.dim, L.norm1, g.pxn, c.dim, c.dim, c.eps, T, stream, pdl));
        DL_TRY(gemmQ40Tc(GEPI_SWIGLU_BF16_, L.w13Qs, L.w13Sc, 2 * c.ffDim, c.dim, g.pxn, c.dim, T, g.phb, c.ffDim, c.numSms, stream, pdl));
        if (tp) {
            arP.parity = 1;
            DL_TRY(gemmQ40Tc(GEPI_STORE_F32_, L.w2Qs, L.w2Sc, c.dim, c.ffDim, g.phb, c.ffDim, T, g.pqkv, c.dim, c.numSms, stream, pdl));
            DL_TRY(launchArResidual(g.px, g.pqkv, c.dim, T, arP, stream, pdl));
        } else DL_TRY(gemmQ40Tc(GEPI_RESIDUAL_, L.w2Qs, L.w2Sc, c.dim, c.ffDim, g.phb, c.ffDim, T, g.px, c.dim, c.numSms, stream, pdl));
    }
    if (wantLogits) {
        GemvArgs a{};
        a.qs = (const uint32_t *)g.wclsQs; a.scales = (const __half *)g.wclsSc; a.d = c.vocab; a.n = c.dim;
        a.normW = g.finalNorm; a.eps = c.eps; a.inStride = c.dim; a.outStride = c.vocab; a.out = g.logits;
        a.in = g.px + (size_t)(T - 1) * c.dim;
        DL_TRY(gemvSel(e, PRO_RMSNORM_, EPI_STORE_, 1, a, c.numSms, stream, false));
    }
    return 0;
}

// Every buffer that only the engine's kernels touch, carved from one zero-filled allocation with the decode step's buffers first
// (one cudaMalloc each decoded 0.5% slower on an H100): the attention, router, MoE, arg-max and prefill counters reset themselves
// and rely on starting at zero.
static bool allocScratch(Engine &e) {
    const EngineConfig &c = e.cfg;
    const size_t mb = c.maxBatch, mp = c.maxPrefill, hd = c.headDim, f = sizeof(float);
    const size_t qDim = c.nHeads * hd, qkvDim = qDim + 2 * c.nKvHeads * hd, kAct = std::max(1u, c.nActiveExperts);
    Buffers &g = e.g;
    size_t off = 0;
    auto carve = [&](auto &p, size_t bytes) {
        p = (std::remove_reference_t<decltype(p)>)((uintptr_t)e.scratch + off);
        off += (bytes + 255) / 256 * 256;
    };
    auto carveAll = [&] {
        off = 0;
        carve(g.qkv, mb * qkvDim * f); carve(g.z, mb * qDim * f); carve(g.h, std::max(mb, kAct) * c.ffDim * f);
        carve(g.attnPartial, mb * c.nHeads * c.nSplits * (hd + 2) * f); carve(g.attnCounters, mb * c.nHeads * 4);
        carve(g.argVal, 256 * f); carve(g.argIdx, 256 * 4); carve(g.argCounter, 16);
        carve(g.expertIdx, mb * kAct * 4); carve(g.expertWeight, mb * kAct * f);
        carve(g.routerLogits, mb * std::max(1u, c.nExperts) * f); carve(g.routerCounter, mb * 4);
        carve(g.moeScratch, kAct * c.dim * f); carve(g.moeCounters, 256 * 4);
        carve(g.pTokens, mp * 4); carve(g.pPos, mp * 4);
        carve(g.px, mp * c.dim * f); carve(g.pqkv, mp * std::max<size_t>(qkvDim, c.dim) * f);   // also the [T][dim] partial of the TP WO / W2 GEMMs
        carve(g.pxn, mp * c.dim * 2); carve(g.pzb, mp * qDim * 2); carve(g.phb, mp * c.ffDim * 2);
        carve(g.pAttnPartial, mp * c.nHeads * (hd + 2) * f); carve(g.pAttnCounters, mp * c.nHeads * 4);
    };
    carveAll();   // sizes
    if (cudaMalloc(&e.scratch, off) != cudaSuccess) return false;
    carveAll();   // pointers
    return cudaMemset(e.scratch, 0, off) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess;   // zero before any client stream runs
}

// Offsets of the symmetric peer-memory arena, every rank alike; returns its size.
static uint64_t arenaLayout(const EngineConfig &c, uint32_t vocabFull, Comm &m) {
    auto align = [](uint64_t x) { return (x + 255) / 256 * 256; };
    const uint64_t N = c.nRanks, mb = c.maxBatch, mp = c.maxPrefill, dim = c.dim;
    m.maxCtas = 256; m.slotStride = c.maxBatch * c.dim; m.prefillSlotStride = c.maxPrefill * c.dim;
    uint64_t off = 0;
    m.slotsOff = off; off = align(off + 2 * N * mb * dim * 8);            // LL words (f32 payload, flag) of the decode all-reduce
    m.flagsOff = off; off = align(off + 2 * N * m.maxCtas * 4);           // logits-gather arrival counters (sampler.cu)
    m.candValOff = off; off = align(off + 8 * 8);                         // cross-rank arg-max candidates, one LL word per rank
    m.gatherOff = off; off = align(off + mb * vocabFull * 4);             // gathered logits (device sampler)
    m.prefillSlotsOff = off; off = align(off + 2 * N * mp * dim * 8);     // LL words of the prefill all-reduce
    return off;
}

static void dropGraph(Engine &e) {
    if (e.decodeGraph) { cudaGraphExecDestroy(e.decodeGraph); e.decodeGraph = nullptr; }
    e.graphGen++;   // round graphs that hold this engine's launches are captured again
}

}  // namespace dl

using dl::Engine;

// rngState: [0] = single-sequence generator, [kChoiceRngSlots + b] = generator of choice b
constexpr uint32_t kChoiceRngSlots = 8;
static_assert(sizeof(Engine::slotLogprobs) == kChoiceRngSlots * sizeof(int), "one logprobs setting per slot");

DL_EXPORT void *dl_engine_create(const dl::EngineConfig *cfg) {
    if (cfg->kvType > 1 || (cfg->kvType == 1 && cfg->headDim % 32)) return nullptr;   // unknown KV-cache storage
    if (cfg->maxPrefill < 1 || cfg->maxPrefill > 256) return nullptr;
    static uint64_t serials = 0;
    Engine *e = new Engine();
    e->cfg = *cfg;
    e->serial = ++serials;
    dl::gHiddenAct = cfg->hiddenAct;
    e->layers.resize(cfg->nLayers);
    e->fusedAttn = std::getenv("DL_NO_FUSED_ATTN") == nullptr;
    e->tcAttn = std::getenv("DL_NO_TC_ATTN") == nullptr;
    if (e->cfg.numSms == 0) {
        int dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        e->cfg.numSms = (uint32_t)sms;
    }
    if (!dl::allocScratch(*e)) {
        dl_engine_destroy(e);
        return nullptr;
    }
    return e;
}

DL_EXPORT void dl_engine_destroy(void *h) {
    Engine *e = (Engine *)h;
    if (!e) return;
    if (e->decodeGraph) cudaGraphExecDestroy(e->decodeGraph);
    if (e->spec) {
        for (cudaGraphExec_t g : e->spec->graph) if (g) cudaGraphExecDestroy(g);
        if (e->spec->dev) cudaFree(e->spec->dev);
        if (e->spec->stage) cudaFreeHost(e->spec->stage);
        delete e->spec;
    }
    if (e->captureStream) cudaStreamDestroy(e->captureStream);
    if (e->megaLayers) cudaFree(e->megaLayers);
    if (e->megaKvScales) cudaFree(e->megaKvScales);
    if (e->megaCounter) cudaFree(e->megaCounter);
    for (void *q : {(void *)e->megaX, (void *)e->megaX2, (void *)e->megaQkv, (void *)e->megaZ, (void *)e->megaH, (void *)e->megaSeq}) if (q) cudaFree(q);
    if (e->abortHost) cudaFreeHost(e->abortHost);
    if (e->ctlCounts) cudaFree(e->ctlCounts);
    if (e->ctlBias) cudaFree(e->ctlBias);
    if (e->slotParams) cudaFree(e->slotParams);
    if (e->slotBias) cudaFree(e->slotBias);
    if (e->slotFiltersDev) cudaFree(e->slotFiltersDev);
    if (e->slotStage) cudaFreeHost(e->slotStage);
    if (e->slotStaged) cudaEventDestroy(e->slotStaged);
    if (e->slotLpDev) cudaFree(e->slotLpDev);
    if (e->slotLpHost) cudaFreeHost(e->slotLpHost);
    if (e->pageDev) cudaFree(e->pageDev);
    if (e->pageHost) cudaFreeHost(e->pageHost);
    if (e->pagesStaged) cudaEventDestroy(e->pagesStaged);
    if (e->scratch) cudaFree(e->scratch);
    delete e;
}

DL_EXPORT int dl_engine_set_layer(void *h, uint32_t layer, const dl::LayerPtrs *p) {
    Engine *e = (Engine *)h;
    if (layer >= e->layers.size()) return -1;
    e->layers[layer] = *p;
    return 0;
}

DL_EXPORT int dl_engine_set_globals(void *h, const dl::GlobalPtrs *p) {
    static_cast<dl::GlobalPtrs &>(((Engine *)h)->g) = *p;
    return 0;
}

// Uploads the per-layer pointer table and switches single-token forwards to the persistent kernel.
DL_EXPORT int dl_engine_enable_mega(void *h, int enable) {
    Engine *e = (Engine *)h;
    if (enable && !e->megaLayers) {
        std::vector<dl::MegaLayer> tab(e->layers.size());
        for (size_t l = 0; l < tab.size(); l++) {
            const dl::LayerPtrs &L = e->layers[l];
            dl::MegaLayer &m = tab[l];
            m.qkvQs = (const uint8_t *)L.qkvQs; m.qkvSc = (const uint8_t *)L.qkvSc; m.woQs = (const uint8_t *)L.woQs; m.woSc = (const uint8_t *)L.woSc;
            m.w13Qs = (const uint8_t *)L.w13Qs; m.w13Sc = (const uint8_t *)L.w13Sc; m.w2Qs = (const uint8_t *)L.w2Qs; m.w2Sc = (const uint8_t *)L.w2Sc;
            m.norm0 = L.norm0; m.norm1 = L.norm1; m.qNorm = L.qNorm; m.kNorm = L.kNorm;
            m.kCache = L.kCache; m.vCache = L.vCache;
        }
        DL_CUDA_CHECK(cudaMalloc(&e->megaLayers, tab.size() * sizeof(dl::MegaLayer)));
        DL_CUDA_CHECK(cudaMemcpy(e->megaLayers, tab.data(), tab.size() * sizeof(dl::MegaLayer), cudaMemcpyHostToDevice));
        if (e->cfg.kvType != 0) {
            std::vector<dl::MegaKvScales> sc(e->layers.size());
            for (size_t l = 0; l < sc.size(); l++) sc[l] = {(__half *)e->layers[l].kScale, (__half *)e->layers[l].vScale};
            DL_CUDA_CHECK(cudaMalloc(&e->megaKvScales, sc.size() * sizeof(dl::MegaKvScales)));
            DL_CUDA_CHECK(cudaMemcpy(e->megaKvScales, sc.data(), sc.size() * sizeof(dl::MegaKvScales), cudaMemcpyHostToDevice));
        }
        DL_CUDA_CHECK(cudaMalloc(&e->megaCounter, 256));
        DL_CUDA_CHECK(cudaMemset(e->megaCounter, 0, 256));
        const dl::EngineConfig &c = e->cfg;
        const size_t qDim = (size_t)c.nHeads * c.headDim, qkvDim = qDim + 2 * (size_t)c.nKvHeads * c.headDim;
        auto allocW = [](uint2 **p, size_t n) {
            const size_t bytes = (n + 8) * sizeof(uint2);
            if (cudaMalloc(p, bytes) != cudaSuccess) return false;
            return cudaMemset(*p, 0, bytes) == cudaSuccess;
        };
        if (!allocW(&e->megaX, c.dim) || !allocW(&e->megaX2, c.dim) || !allocW(&e->megaQkv, qkvDim) || !allocW(&e->megaZ, qDim) || !allocW(&e->megaH, c.ffDim)) return -41;
        DL_CUDA_CHECK(cudaMalloc(&e->megaSeq, 256));
        const unsigned int one = 1;
        DL_CUDA_CHECK(cudaMemset(e->megaSeq, 0, 256));
        DL_CUDA_CHECK(cudaMemcpy(e->megaSeq, &one, sizeof(one), cudaMemcpyHostToDevice));   // epochs start at 1024: never equal to the zeroed words
        if (!e->abortHost) {
            DL_CUDA_CHECK(cudaHostAlloc((void **)&e->abortHost, 64, cudaHostAllocMapped));
            std::memset(e->abortHost, 0, 64);
            DL_CUDA_CHECK(cudaHostGetDevicePointer((void **)&e->abortDev, e->abortHost, 0));
        }
        if (const char *g = std::getenv("DL_MEGA_CTAS")) e->megaCtas = (uint32_t)std::atoi(g);
        if (const char *g = std::getenv("DL_MEGA_FLAGS")) e->megaFlags = (uint32_t)std::atoi(g);
        if (const char *g = std::getenv("DL_MEGA_INFLIGHT")) e->megaInflight = (uint32_t)std::atoi(g);
    }
    e->useMega = enable != 0;
    dl::dropGraph(*e);   // the captured step runs the kernels chosen at capture
    return 0;
}

DL_EXPORT int dl_engine_set_vocab_limit(void *h, uint32_t limit) {
    Engine *e = (Engine *)h;
    if (e->vocabLimit != limit) dl::dropGraph(*e);   // the limit is baked into the captured launch
    e->vocabLimit = limit;
    return 0;
}

// Nanoseconds the persistent kernel (CTA 0) has spent waiting for peer ranks inside the fused all-reduce epilogues since engine
// creation (host-mapped counter: readable without a device synchronisation; exact after the stream has been synchronised).
DL_EXPORT unsigned long long dl_engine_sync_ns(void *h) {
    Engine *e = (Engine *)h;
    unsigned long long v = 0;
    if (e->megaSeq && cudaMemcpy(&v, e->megaSeq + 2, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return 0ull;
    return v;
}

// 1 when a device-side wait loop gave up (dead peer rank, CTA that never became resident): the results of that step are invalid.
DL_EXPORT int dl_engine_aborted(void *h) {
    Engine *e = (Engine *)h;
    return (e->abortHost && *e->abortHost) ? 1 : 0;
}

// Seeds the device-resident xorshift* generator (same stream of coins as the host Sampler for the same seed) and allocates the
// sampler scratch. Under tensor parallelism every rank must call this with the same seed.
static int ensureSampler(Engine *e) {
    const dl::EngineConfig &c = e->cfg;
    if (!e->rngState) {
        DL_CUDA_CHECK(cudaMalloc(&e->rngState, 2 * kChoiceRngSlots * sizeof(unsigned long long)));
        DL_CUDA_CHECK(cudaMalloc(&e->probScratch, ((size_t)c.maxBatch * c.vocab * (c.nRanks ? c.nRanks : 1) + 16) * sizeof(float)));
        DL_CUDA_CHECK(cudaMalloc(&e->gatherEpoch, 64));
        DL_CUDA_CHECK(cudaMemset(e->gatherEpoch, 0, 64));
        DL_CUDA_CHECK(cudaMalloc(&e->gatherBlockCounter, 64));
        DL_CUDA_CHECK(cudaMemset(e->gatherBlockCounter, 0, 64));
        if (e->comm.nRanks > 1) {
            float *g[dl::kApiMaxRanks] = {};
            unsigned int *f[dl::kApiMaxRanks] = {};
            for (uint32_t r = 0; r < e->comm.nRanks; r++) {
                g[r] = (float *)((uint8_t *)e->comm.arena[r] + e->comm.gatherOff);
                f[r] = (unsigned int *)((uint8_t *)e->comm.arena[r] + e->comm.flagsOff);
            }
            DL_CUDA_CHECK(cudaMalloc(&e->gatherUcDev, sizeof(g)));
            DL_CUDA_CHECK(cudaMalloc(&e->flagUcDev, sizeof(f)));
            DL_CUDA_CHECK(cudaMemcpy(e->gatherUcDev, g, sizeof(g), cudaMemcpyHostToDevice));
            DL_CUDA_CHECK(cudaMemcpy(e->flagUcDev, f, sizeof(f), cudaMemcpyHostToDevice));
        }
    }
    return 0;
}

// Count rows [1 + kChoiceRngSlots][vocabFull] of the sampling controls (row 0: single sequence, row 1 + b: choice or slot b).
static int ensureCounts(Engine *e, cudaStream_t stream) {
    const uint32_t full = e->cfg.vocab * (e->comm.nRanks > 1 ? e->comm.nRanks : 1);
    const size_t bytes = (size_t)(1 + kChoiceRngSlots) * full * sizeof(uint32_t);
    if (!e->ctlCounts) {
        DL_CUDA_CHECK(cudaMalloc(&e->ctlCounts, bytes));
        DL_CUDA_CHECK(cudaMemsetAsync(e->ctlCounts, 0, bytes, stream));
    }
    return 0;
}

// Paged slots: copies the host page table to the device on `stream` if it changed since the last upload.
static int uploadPages(Engine *e, cudaStream_t stream) {
    if (!e->pagesDirty) return 0;
    DL_CUDA_CHECK(cudaMemcpyAsync(e->pageDev, e->pageHost, (size_t)kChoiceRngSlots * e->nPages * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaEventRecord(e->pagesStaged, stream));
    e->pagesDirty = false;
    return 0;
}

// Paged slots: the host page table may be rewritten once the last upload has read it.
static int editPages(Engine *e) {
    DL_CUDA_CHECK(cudaEventSynchronize(e->pagesStaged));
    e->pagesDirty = true;
    return 0;
}

DL_EXPORT int dl_engine_sampler_seed(void *h, unsigned long long seed) {
    Engine *e = (Engine *)h;
    DL_TRY(ensureSampler(e));
    if (seed == 0) seed = 0x9E3779B97F4A7C15ull;   // xorshift state must not be zero
    DL_CUDA_CHECK(cudaMemcpy(e->rngState, &seed, sizeof(seed), cudaMemcpyHostToDevice));
    return 0;
}

// Current state of the single-sequence generator (0 before the first seeding). Seeding with it continues the same stream.
DL_EXPORT unsigned long long dl_engine_sampler_state(void *h) {
    Engine *e = (Engine *)h;
    unsigned long long v = 0;
    if (e->rngState && cudaMemcpy(&v, e->rngState, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return 0ull;
    return v;
}

// The sampling controls of the following draws: presence and frequency penalties and a logit bias given as nBias (id, value) pairs
// (ids in [0, V), V = the sampled vocabulary). Zeroes the count rows set in rowMask (bit 0: single sequence, bit 1 + b: choice b),
// so call it at the start of every completion. All zero (and no bias) switches the controls off: the draws are exactly those
// without controls. Under tensor parallelism every rank makes the same call and keeps identical counts. The uploads run on `stream`
// (the stream of the draws) and are complete when the call returns.
DL_EXPORT int dl_engine_set_sampling_controls(void *h, float presence, float frequency, const int32_t *ids, const float *vals, int nBias,
                                              uint32_t rowMask, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    const uint32_t full = e->cfg.vocab * (e->comm.nRanks > 1 ? e->comm.nRanks : 1);
    const uint32_t n = (e->vocabLimit && e->vocabLimit < full) ? e->vocabLimit : full;
    const uint32_t rows = 1 + kChoiceRngSlots;
    if (nBias < 0 || (rowMask >> rows) != 0) return -52;
    for (int i = 0; i < nBias; i++) if (ids[i] < 0 || (uint32_t)ids[i] >= n) return -53;
    e->ctlActive = false;   // set again only once every buffer below is in place
    if (presence == 0.f && frequency == 0.f && nBias == 0) return 0;
    DL_TRY(ensureSampler(e));
    DL_TRY(ensureCounts(e, stream));
    if (!e->ctlBias) DL_CUDA_CHECK(cudaMalloc(&e->ctlBias, (size_t)full * sizeof(float)));
    std::vector<float> bias;
    if (nBias > 0) {
        bias.assign(full, 0.f);
        for (int i = 0; i < nBias; i++) bias[ids[i]] = vals[i];
        DL_CUDA_CHECK(cudaMemcpyAsync(e->ctlBias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    }
    for (uint32_t r = 0; r < rows; r++)
        if ((rowMask >> r) & 1u) DL_CUDA_CHECK(cudaMemsetAsync(e->ctlCounts + (size_t)r * full, 0, (size_t)full * sizeof(uint32_t), stream));
    DL_CUDA_CHECK(cudaStreamSynchronize(stream));   // `bias` is a host temporary
    e->ctlPresence = presence;
    e->ctlFrequency = frequency;
    e->ctlBiasActive = nBias > 0;
    e->ctlActive = true;
    return 0;
}

// The active controls for draws whose row 0 uses count row `firstRow` (null: none).
static const dl::SampleControls *activeControls(const Engine *e, uint32_t firstRow, dl::SampleControls &ctl) {
    if (!e->ctlActive) return nullptr;
    const uint32_t full = e->cfg.vocab * (e->comm.nRanks > 1 ? e->comm.nRanks : 1);
    ctl = dl::SampleControls{e->ctlBiasActive ? e->ctlBias : nullptr, e->ctlCounts + (size_t)firstRow * full, full, e->ctlPresence, e->ctlFrequency};
    return &ctl;
}

static bool filtersOn(const dl::SampleFilters &f) { return f.topK > 0 || f.minP > 0.f; }

// The sampling filters (kernels.h: SampleFilters) of the following sampled draws of the single sequence (dl_engine_sample) and of
// the choices (dl_engine_sample_rows): topK 0 and minP 0 switch them off. They persist until changed. Temperature-0 draws ignore
// them. Under tensor parallelism every rank makes the same call.
DL_EXPORT int dl_engine_set_sampling_filters(void *h, uint32_t topK, float minP) {
    Engine *e = (Engine *)h;
    const dl::SampleFilters f{topK, minP};
    if (!dl::sampleFiltersValid(f)) return -54;
    e->filters = f;
    return 0;
}

// Samples the next token from the logits of the last forward (logitsMode 1) on the device: tokens[0] <- sample, pos[0]++, history.
// Tensor parallel: the vocabulary slices are first gathered into every rank's arena (peer / multicast stores, no NCCL); every rank
// then draws the same token from its own copy of the generator. With sampling controls active, temperature 0 draws the arg-max of
// the controlled logits.
DL_EXPORT int dl_engine_sample(void *h, float temperature, float topp, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    const dl::EngineConfig &c = e->cfg;
    if (!e->rngState) return -50;
    const uint32_t nR = e->comm.nRanks > 1 ? e->comm.nRanks : 1;
    const uint32_t full = c.vocab * nR;
    const uint32_t n = (e->vocabLimit && e->vocabLimit < full) ? e->vocabLimit : full;
    dl::SampleControls ctlArgs;
    const dl::SampleControls *ctl = activeControls(e, 0, ctlArgs);
    const dl::SampleFilters *filt = filtersOn(e->filters) ? &e->filters : nullptr;
    if (nR == 1)
        return dl::launchSample(e->g.logits, e->probScratch, n, temperature, topp, e->rngState, e->g.tokens, e->g.pos, e->g.history, c.seqLen,
                                nullptr, nullptr, 1, stream, ctl, filt);
    uint8_t *mine = (uint8_t *)e->comm.arena[e->comm.rank];
    float *gatherLocal = (float *)(mine + e->comm.gatherOff);
    unsigned int *flagLocal = (unsigned int *)(mine + e->comm.flagsOff);
    float *gatherMc = e->comm.mcArena ? (float *)((uint8_t *)e->comm.mcArena + e->comm.gatherOff) : nullptr;
    unsigned int *flagMc = e->comm.mcArena ? (unsigned int *)((uint8_t *)e->comm.mcArena + e->comm.flagsOff) : nullptr;
    DL_TRY(dl::launchLogitsGather(e->g.logits, c.vocab, c.rank, nR, gatherMc, e->gatherUcDev, flagMc, e->flagUcDev, e->gatherBlockCounter, stream));
    return dl::launchSample(gatherLocal, e->probScratch, n, temperature, topp, e->rngState, e->g.tokens, e->g.pos, e->g.history, c.seqLen, flagLocal,
                            e->gatherEpoch, nR, stream, ctl, filt);
}

// Seeds the n <= 8 generators of the batched sampler. They are separate from the single-sequence generator of dl_engine_sample,
// which keeps its stream. Every rank must pass the same seeds.
DL_EXPORT int dl_engine_sampler_seed_rows(void *h, const unsigned long long *seeds, int n) {
    Engine *e = (Engine *)h;
    if (n < 1 || n > (int)kChoiceRngSlots) return -51;
    DL_TRY(ensureSampler(e));
    unsigned long long s[kChoiceRngSlots];
    for (int i = 0; i < n; i++) s[i] = seeds[i] ? seeds[i] : 0x9E3779B97F4A7C15ull;
    DL_CUDA_CHECK(cudaMemcpy(e->rngState + kChoiceRngSlots, s, n * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    return 0;
}

// nb draws into tokens[0..nb), row b with batched-sampler generator b. firstStep: every row draws from the logits row of the last single-token
// forward (logits[0]); otherwise row b draws from logits[b] of a choices forward. Rows set in inactiveMask draw nothing.
// Tensor parallel: the vocabulary slices of the rows are gathered first and every rank draws the same tokens.
DL_EXPORT int dl_engine_sample_rows(void *h, int nb, uint32_t inactiveMask, float temperature, float topp, int firstStep, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    const dl::EngineConfig &c = e->cfg;
    if (!e->rngState) return -50;
    if (nb < 1 || (uint32_t)nb > c.maxBatch || nb > (int)kChoiceRngSlots) return -10;
    const uint32_t nR = e->comm.nRanks > 1 ? e->comm.nRanks : 1;
    const uint32_t full = c.vocab * nR;
    const uint32_t n = (e->vocabLimit && e->vocabLimit < full) ? e->vocabLimit : full;
    const uint32_t rows = firstStep ? 1u : (uint32_t)nb;
    dl::SampleControls ctlArgs;
    const dl::SampleControls *ctl = activeControls(e, 1, ctlArgs);
    const dl::SampleFilters *filt = filtersOn(e->filters) ? &e->filters : nullptr;
    if (nR == 1)
        return dl::launchSampleRows(e->g.logits, firstStep ? 0u : c.vocab, e->probScratch, n, temperature, topp, e->rngState + kChoiceRngSlots, e->g.tokens, nb,
                                    inactiveMask, nullptr, nullptr, 1, stream, ctl, nullptr, filt);
    uint8_t *mine = (uint8_t *)e->comm.arena[e->comm.rank];
    float *gatherLocal = (float *)(mine + e->comm.gatherOff);
    unsigned int *flagLocal = (unsigned int *)(mine + e->comm.flagsOff);
    float *gatherMc = e->comm.mcArena ? (float *)((uint8_t *)e->comm.mcArena + e->comm.gatherOff) : nullptr;
    unsigned int *flagMc = e->comm.mcArena ? (unsigned int *)((uint8_t *)e->comm.mcArena + e->comm.flagsOff) : nullptr;
    DL_TRY(dl::launchLogitsGather(e->g.logits, c.vocab, c.rank, nR, gatherMc, e->gatherUcDev, flagMc, e->flagUcDev, e->gatherBlockCounter, stream, rows));
    return dl::launchSampleRows(gatherLocal, firstStep ? 0u : full, e->probScratch, n, temperature, topp, e->rngState + kChoiceRngSlots, e->g.tokens, nb, inactiveMask,
                                flagLocal, e->gatherEpoch, nR, stream, ctl, nullptr, filt);
}

// Log-probabilities of the tokens the last step drew (logprobs.cu), enqueued on `stream` behind the draw: row b of the last
// forward's logits (every row reads logits[0] with kLogprobsSharedRow: the choices' first draw) and the token in tokens[b], for
// the rows set in rowMask (b < rows), with k[b] (host, 0..20) top entries. kLogprobsControlled: the logits are transformed by the
// sampling controls the draw used, with count row firstRow + b (0: single sequence, 1 + b: choice b). out: device int32
// [rows][kLogprobsWords]. Single GPU only. flags: dl::kLogprobsControlled, dl::kLogprobsSharedRow (engine_api.h).

DL_EXPORT int dl_engine_logprobs(void *h, int rows, uint32_t rowMask, const int32_t *k, int firstRow, int flags, int32_t *out, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    const dl::EngineConfig &c = e->cfg;
    if (e->comm.nRanks > 1) return -70;
    if (rows < 1 || (uint32_t)rows > c.maxBatch || firstRow < 0 || (uint32_t)(firstRow + rows) > 1 + kChoiceRngSlots) return -10;
    dl::SampleControls ctlArgs;
    const dl::SampleControls *ctl = (flags & dl::kLogprobsControlled) ? activeControls(e, (uint32_t)firstRow, ctlArgs) : nullptr;
    return dl::launchLogprobsRows(e->g.logits, (flags & dl::kLogprobsSharedRow) ? 0u : c.vocab, dl::localVocabLimit(*e), (uint32_t)rows, rowMask, k,
                                  e->g.tokens, out, stream, ctl);
}

DL_EXPORT uint64_t dl_engine_arena_bytes(void *h) {
    dl::Comm layout{};
    return dl::arenaLayout(((Engine *)h)->cfg, ((Engine *)h)->g.vocabFull, layout);
}

// Every rank's arena of dl_engine_arena_bytes bytes, zeroed on every rank before any rank's kernels use it.
DL_EXPORT int dl_engine_set_comm(void *h, const dl::CommPtrs *p) {
    Engine *e = (Engine *)h;
    if (p->nRanks != e->cfg.nRanks) return -2;
    static_cast<dl::CommPtrs &>(e->comm) = *p;
    dl::arenaLayout(e->cfg, e->g.vocabFull, e->comm);
    return 0;
}

DL_EXPORT int dl_engine_set_trace(void *h, uint64_t *buf, uint32_t capLaunches) {
    ((Engine *)h)->trace = buf;
    ((Engine *)h)->traceCap = capLaunches;
    dl::dropGraph(*(Engine *)h);   // the trace buffer is a launch parameter of the captured step
    return 0;
}

DL_EXPORT int dl_engine_set_trace_all(void *h, int allCtas) {
    ((Engine *)h)->traceAllCtas = allCtas != 0;
    dl::dropGraph(*(Engine *)h);
    return 0;
}

DL_EXPORT int dl_engine_mega_active(void *h) { return ((Engine *)h)->lastDecodeMega ? 1 : 0; }

// Copies the persistent kernel's phase vectors, 8 zeroed tail words included, into caller-provided device memory: x (dim + 8
// LL words), q|k|v (qkvDim + 8 LL words), z (qDim + 8 LL words) and the SwiGLU output (ffDim plain f32 in a buffer of ffDim + 8
// words). Changes no engine state. -1 before the first dl_engine_enable_mega.
DL_EXPORT int dl_engine_mega_copy_vectors(void *h, void *x, void *qkv, void *z, void *hF, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    if (!e->megaX) return -1;
    const dl::EngineConfig &c = e->cfg;
    const size_t qDim = (size_t)c.nHeads * c.headDim, qkvDim = qDim + 2 * (size_t)c.nKvHeads * c.headDim;
    void *dst[4] = {x, qkv, z, hF};
    const uint2 *src[4] = {e->megaX, e->megaQkv, e->megaZ, e->megaH};
    const size_t n[4] = {c.dim, qkvDim, qDim, c.ffDim};
    for (int i = 0; i < 4; i++) DL_CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], (n[i] + 8) * sizeof(uint2), cudaMemcpyDeviceToDevice, stream));
    return 0;
}

DL_EXPORT uint32_t dl_engine_num_sms(void *h) { return ((Engine *)h)->cfg.numSms; }

DL_EXPORT int dl_engine_forward(void *h, int nb, int logitsMode, int greedyAdvance, cudaStream_t stream) {
    return dl::engineForward(*(Engine *)h, nb, logitsMode, greedyAdvance != 0, stream);
}

// Library-collective building blocks (decode path, nb tokens): the same kernels, but the tensor-parallel partial products
// are *stored* into `ybuf` instead of being all-reduced in the epilogue; the caller all-reduces ybuf with NCCL and adds it
// to x. Used (a) as the NCCL baseline the fused kernels are measured against, (b) as the execution path when ranks do not
// share an NVLink/IPC domain (multi-node) and (c) for dense f32/f16 weight files under tensor parallelism.
//   part 0: embedding              part 1: QKV + attention + WO -> ybuf
//   part 2: feed-forward -> ybuf   part 3: logits of the last token (local vocabulary slice)   part 4: logits of all nb tokens
DL_EXPORT int dl_engine_forward_part(void *h, int nb, uint32_t layer, int part, float *ybuf, cudaStream_t stream) {
    Engine &e = *(Engine *)h;
    const dl::EngineConfig &c = e.cfg;
    const uint32_t qDim = c.nHeads * c.headDim, kvDim = c.nKvHeads * c.headDim, qkvDim = qDim + 2 * kvDim;
    if (nb < 1 || (uint32_t)nb > c.maxBatch || (nb & (nb - 1))) return -10;
    if (part == 0) return dl::launchEmbedding(embTable(e), e.g.tokens, e.g.x, c.dim, c.dim, e.g.vocabFull, nb, stream);
    if (part == 3 || part == 4) {
        dl::GemvArgs a{};
        a.qs = (const uint32_t *)e.g.wclsQs; a.scales = (const __half *)e.g.wclsSc; a.d = c.vocab; a.n = c.dim;
        a.normW = e.g.finalNorm; a.eps = c.eps; a.inStride = c.dim; a.outStride = c.vocab; a.out = e.g.logits;
        a.in = part == 3 ? e.g.x + (size_t)(nb - 1) * c.dim : e.g.x;
        return dl::gemvSel(e, dl::PRO_RMSNORM_, dl::EPI_STORE_, part == 3 ? 1 : nb, a, c.numSms, stream, false);
    }
    if (layer >= c.nLayers) return -1;
    const dl::LayerPtrs &L = e.layers[layer];
    dl::GemvArgs a{};
    if (part == 1) {
        a.qs = (const uint32_t *)L.qkvQs; a.scales = (const __half *)L.qkvSc; a.d = qkvDim; a.n = c.dim;
        a.in = e.g.x; a.inStride = c.dim; a.normW = L.norm0; a.eps = c.eps; a.out = e.g.qkv; a.outStride = qkvDim;
        DL_TRY(dl::gemvSel(e, dl::PRO_RMSNORM_, dl::EPI_STORE_, nb, a, c.numSms, stream, false));
        const dl::RopeKvArgs r = dl::layerRopeKv(e, L, e.g.qkv, e.g.pos, 0, c.seqLen);
        DL_TRY(dl::launchRopeKv(r, nb, stream, false));
        dl::AttnArgs t{};
        t.qkv = e.g.qkv; t.qkvStride = qkvDim; t.pos = e.g.pos; t.kCache = r.kCache; t.vCache = r.vCache; t.kScale = r.kScale; t.vScale = r.vScale;
        t.nHeads = c.nHeads; t.nKvHeads = c.nKvHeads; t.headDim = c.headDim; t.seqLen = c.seqLen; t.nSplits = c.nSplits;
        t.partial = e.g.attnPartial; t.counters = e.g.attnCounters; t.out = e.g.z; t.outStride = qDim;
        DL_TRY(dl::launchAttnDecode(t, nb, stream, false));
        a = dl::GemvArgs{};
        a.qs = (const uint32_t *)L.woQs; a.scales = (const __half *)L.woSc; a.d = c.dim; a.n = qDim;
        a.in = e.g.z; a.inStride = qDim; a.out = ybuf; a.outStride = c.dim;
        return dl::gemvSel(e, dl::PRO_PLAIN_, dl::EPI_STORE_, nb, a, c.numSms, stream, false);
    }
    if (part == 2 && c.nExperts > 0) {
        if (nb != 1) return -13;
        DL_CUDA_CHECK(cudaMemsetAsync(ybuf, 0, (size_t)c.dim * sizeof(float), stream));
        return dl::runMoe(e, L, ybuf, false, nullptr, nullptr, stream, false);
    }
    if (part == 2) {
        a.qs = (const uint32_t *)L.w13Qs; a.scales = (const __half *)L.w13Sc; a.d = 2 * c.ffDim; a.n = c.dim;
        a.in = e.g.x; a.inStride = c.dim; a.normW = L.norm1; a.eps = c.eps; a.out = e.g.h; a.outStride = c.ffDim;
        DL_TRY(dl::gemvSel(e, dl::PRO_RMSNORM_, dl::EPI_SWIGLU_, nb, a, c.numSms, stream, false));
        a = dl::GemvArgs{};
        a.qs = (const uint32_t *)L.w2Qs; a.scales = (const __half *)L.w2Sc; a.d = c.dim; a.n = c.ffDim;
        a.in = e.g.h; a.inStride = c.ffDim; a.out = ybuf; a.outStride = c.dim;
        return dl::gemvSel(e, dl::PRO_PLAIN_, dl::EPI_STORE_, nb, a, c.numSms, stream, false);
    }
    return -2;
}

// One choices step: nb (power of two, <= maxBatch) tokens staged in tokens[0..nb) with pos[0..nb) = P + 1 + j. Row b attends to
// the prompt rows [0, P] and its own rows [P + 1 + b * C, P + 1 + b * C + j] and appends its K/V at P + 1 + b * C + j; rows set
// in inactiveMask (finished choices, batch padding) write no K/V. Logits of all nb rows land in logits[0..nb).
DL_EXPORT int dl_engine_choices_forward(void *h, int nb, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, cudaStream_t stream) {
    const dl::ChoiceStep ch{P, C, j, inactiveMask};
    return dl::engineForward(*(Engine *)h, nb, 2, false, stream, &ch);
}

// Decode mixture-of-experts feed-forward of one token on one rank (tests/test_gpu_moe.py): the engine's launch sequence with the
// caller's buffers (see MoeDecodeArgs) and the gate activation passed explicitly (0 = SiLU, 1 = GELU). No programmatic dependent launch.
DL_EXPORT int dl_moe_decode_ffn(const float *x, float *out, const float *norm, const float *gate, const void *w13Qs, const void *w13Sc,
                                const void *w2Qs, const void *w2Sc, uint32_t dim, uint32_t ff, uint32_t nExperts, uint32_t k,
                                uint32_t firstLocal, uint32_t nLocal, float eps, float *routerLogits, unsigned int *routerCounter,
                                int *expertIdx, float *expertWeight, float *hOut, float *moeScratch, unsigned int *moeCounters,
                                uint32_t numSms, uint32_t hiddenAct, cudaStream_t stream) {
    dl::MoeDecodeArgs m{};
    m.x = x; m.out = out; m.norm = norm; m.gate = gate; m.w13Qs = w13Qs; m.w13Sc = w13Sc; m.w2Qs = w2Qs; m.w2Sc = w2Sc;
    m.dim = dim; m.ff = ff; m.nExperts = nExperts; m.k = k; m.firstLocal = firstLocal; m.nLocal = nLocal; m.eps = eps;
    m.routerLogits = routerLogits; m.routerCounter = routerCounter; m.expertIdx = expertIdx; m.expertWeight = expertWeight;
    m.h = hOut; m.moeScratch = moeScratch; m.moeCounters = moeCounters; m.numSms = numSms;
    const dl::HiddenActScope act(hiddenAct);
    return dl::moeDecodeFfn(m, stream, false);
}

// dl_moe_decode_ffn for dense experts (tests/test_gpu_moe_dense.py): wtype 1 = f32, 2 = f16; w13 is [nLocal][2 * ff][dim] with
// gate and up rows interleaved, w2 is [nLocal][dim][ff].
DL_EXPORT int dl_moe_decode_ffn_dense(int wtype, const float *x, float *out, const float *norm, const float *gate, const void *w13,
                                      const void *w2, uint32_t dim, uint32_t ff, uint32_t nExperts, uint32_t k, uint32_t firstLocal,
                                      uint32_t nLocal, float eps, float *routerLogits, unsigned int *routerCounter, int *expertIdx,
                                      float *expertWeight, float *hOut, float *moeScratch, unsigned int *moeCounters, uint32_t numSms,
                                      uint32_t hiddenAct, cudaStream_t stream) {
    if (wtype != 1 && wtype != 2) return -4;
    dl::MoeDecodeArgs m{};
    m.x = x; m.out = out; m.norm = norm; m.gate = gate; m.w13Qs = w13; m.w2Qs = w2; m.wType = wtype;
    m.dim = dim; m.ff = ff; m.nExperts = nExperts; m.k = k; m.firstLocal = firstLocal; m.nLocal = nLocal; m.eps = eps;
    m.routerLogits = routerLogits; m.routerCounter = routerCounter; m.expertIdx = expertIdx; m.expertWeight = expertWeight;
    m.h = hOut; m.moeScratch = moeScratch; m.moeCounters = moeCounters; m.numSms = numSms;
    const dl::HiddenActScope act(hiddenAct);
    return dl::moeDecodeFfn(m, stream, false);
}

namespace dl {

struct PrefillChunk { uint32_t T, p0, onTc; };

// The chunks of a prompt of n tokens at positions p0 .. p0 + n - 1 in a cache of `rows` rows. A chunk of up to maxPrefill tokens
// runs on the tensor cores while at least minTc (0: never) tokens remain and tcAllowed; otherwise the largest power-of-two GEMV
// batch <= min(remaining, maxBatch) runs. slot >= 0 (a KV-cache slot of `slots`): every chunk on the tensor cores.
// -64: slot prefill without slots; -60: the prompt runs past the cache.
static int planPrefill(uint32_t n, uint32_t p0, int slot, uint32_t slots, uint32_t rows, uint32_t maxPrefill, uint32_t maxBatch,
                       uint32_t minTc, bool tcAllowed, std::vector<PrefillChunk> &out) {
    out.clear();
    if (slot >= 0 && slots < 2) return -64;
    if ((uint64_t)p0 + n > rows) return -60;
    if (maxPrefill < 1) return -11;
    const bool tc = minTc > 0 && tcAllowed;
    for (uint32_t i = 0; i < n;) {
        const uint32_t rem = n - i;
        const bool onTc = slot >= 0 || (tc && rem >= minTc);
        uint32_t T = 1;
        if (onTc) T = std::min(rem, maxPrefill);
        else while (T * 2 <= std::min(rem, maxBatch)) T *= 2;
        out.push_back({T, p0 + i, onTc ? 1u : 0u});
        i += T;
    }
    return 0;
}

// planPrefill with the engine's settings. The tensor cores take q40 matrices; MoE: dim and ff multiples of 256 (grouped GEMMs);
// tensor parallel: per-rank qDim, ff and dim multiples of 256 (prefill all-reduce).
static int planEnginePrefill(const Engine &e, uint32_t n, uint32_t p0, int slot, std::vector<PrefillChunk> &out) {
    const EngineConfig &c = e.cfg;
    const bool tpOk = e.comm.nRanks <= 1 || ((c.nHeads * c.headDim) % 256 == 0 && c.ffDim % 256 == 0 && c.dim % 256 == 0);
    const bool moeOk = c.nExperts == 0 || (c.dim % 256 == 0 && c.ffDim % 256 == 0);
    return planPrefill(n, p0, slot, e.slots, slot >= 0 ? e.slotLen : c.seqLen, c.maxPrefill, c.maxBatch, e.prefillMinTc,
                       c.wType == 0 && tpOk && moeOk, out);
}

static int copyPlan(int rc, const std::vector<PrefillChunk> &chunks, uint32_t *out, uint32_t cap) {
    if (rc != 0) return rc;
    for (size_t i = 0; i < chunks.size() && i < cap; i++) {
        out[3 * i] = chunks[i].T; out[3 * i + 1] = chunks[i].p0; out[3 * i + 2] = chunks[i].onTc;
    }
    return (int)chunks.size();
}

}  // namespace dl

// The prefill schedule without an engine or a device (see planPrefill): writes up to `cap` chunks as (T, p0, on tensor cores)
// triples and returns the number of chunks, or a negative error.
DL_EXPORT int dl_prefill_plan(uint32_t n, uint32_t p0, int slot, uint32_t slots, uint32_t rows, uint32_t maxPrefill, uint32_t maxBatch,
                              uint32_t minTc, int tcAllowed, uint32_t *out, uint32_t cap) {
    std::vector<dl::PrefillChunk> chunks;
    return dl::copyPlan(dl::planPrefill(n, p0, slot, slots, rows, maxPrefill, maxBatch, minTc, tcAllowed != 0, chunks), chunks, out, cap);
}

// The chunks dl_engine_prefill runs for these arguments, as dl_prefill_plan returns them.
DL_EXPORT int dl_engine_prefill_plan(void *h, uint32_t n, uint32_t p0, int slot, uint32_t *out, uint32_t cap) {
    std::vector<dl::PrefillChunk> chunks;
    return dl::copyPlan(dl::planEnginePrefill(*(Engine *)h, n, p0, slot, chunks), chunks, out, cap);
}

// A prompt of n tokens (host memory) at positions p0 .. p0 + n - 1, staged chunk by chunk (planEnginePrefill) on `stream`;
// logits of the last token with wantLogits. slot >= 0: into KV-cache slot `slot`.
DL_EXPORT int dl_engine_prefill(void *h, const int32_t *hostTokens, uint32_t n, uint32_t p0, int slot, int wantLogits, cudaStream_t stream) {
    Engine &e = *(Engine *)h;
    std::vector<dl::PrefillChunk> chunks;
    DL_TRY(dl::planEnginePrefill(e, n, p0, slot, chunks));
    if (slot >= 0 && e.pagedSlots) {
        if ((uint64_t)p0 + n > (uint64_t)e.slotPages[slot] * dl::kPageRows) return -60;   // reserve the rows first (dl_engine_slot_reserve)
        DL_TRY(uploadPages(&e, stream));
    }
    std::vector<int32_t> pos(n);
    for (uint32_t i = 0; i < n; i++) pos[i] = (int32_t)(p0 + i);
    for (const dl::PrefillChunk &ch : chunks) {
        const uint32_t i = ch.p0 - p0, T = ch.T;
        const bool logits = wantLogits && i + T == n;
        // pageable sources: each copy has read its host bytes when the call returns
        DL_CUDA_CHECK(cudaMemcpyAsync(ch.onTc ? e.g.pTokens : e.g.tokens, hostTokens + i, T * 4, cudaMemcpyHostToDevice, stream));
        DL_CUDA_CHECK(cudaMemcpyAsync(ch.onTc ? e.g.pPos : e.g.pos, pos.data() + i, T * 4, cudaMemcpyHostToDevice, stream));
        if (ch.onTc) DL_TRY(dl::enginePrefill(e, T, ch.p0, logits, stream, slot));
        else DL_TRY(dl::engineForward(e, (int)T, logits ? 1 : 0, false, stream));
    }
    return 0;
}

// Copies the intermediates the last prompt chunk left in the engine's scratch into caller device memory (tests), `rows` rows
// each; a null destination is skipped. Tensor-core chunk (rows <= maxPrefill): px (f32 [rows][dim], the residual), pqkv (f32
// [rows][qkvDim], q after QK-norm and RoPE, raw k and v), pxn (bf16 [rows][dim], the last rmsnorm), pzb (bf16 [rows][qDim],
// attention) and phb (bf16 [rows][ff], SwiGLU). GEMV batch (rows <= maxBatch): qkv (f32 [rows][qkvDim]), z (f32 [rows][qDim],
// attention) and hF (f32 [rows][ff], SwiGLU); the residual is the client's x. Every buffer holds the last layer's values.
DL_EXPORT int dl_engine_prefill_scratch(void *h, uint32_t rows, void *px, void *pqkv, void *pxn, void *pzb, void *phb, void *qkv,
                                        void *z, void *hF, cudaStream_t stream) {
    Engine &e = *(Engine *)h;
    const dl::EngineConfig &c = e.cfg;
    const size_t qDim = (size_t)c.nHeads * c.headDim, qkvDim = qDim + 2 * (size_t)c.nKvHeads * c.headDim;
    if ((px || pqkv || pxn || pzb || phb) && rows > c.maxPrefill) return -1;
    if ((qkv || z || hF) && rows > c.maxBatch) return -1;
    void *dst[8] = {px, pqkv, pxn, pzb, phb, qkv, z, hF};
    const void *src[8] = {e.g.px, e.g.pqkv, e.g.pxn, e.g.pzb, e.g.phb, e.g.qkv, e.g.z, e.g.h};
    const size_t bytes[8] = {c.dim * 4, qkvDim * 4, c.dim * 2, qDim * 2, (size_t)c.ffDim * 2, qkvDim * 4, qDim * 4, (size_t)c.ffDim * 4};
    for (int i = 0; i < 8; i++)
        if (dst[i]) DL_CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], rows * bytes[i], cudaMemcpyDeviceToDevice, stream));
    return 0;
}

// The mixture-of-experts stages of the last prompt chunk's last layer (tests), a null destination skipped. Tensor-core chunk of
// `rows` tokens (the process-wide MoE prefill scratch; -1 unless its last call had this engine's shape and `rows` tokens): router logits f32
// [rows][nExperts], expert ids and weights [rows][k], and the SwiGLU output of every (token, slot) pair, bf16 [rows][k][ff]. One-token
// step (rows = 1): router logits [nExperts], ids and weights [k], and h f32 [k][ff]. The MoE rmsnorm output and the residual are
// those of dl_engine_prefill_scratch.
DL_EXPORT int dl_engine_moe_scratch(void *h, uint32_t rows, int tensorCores, void *logits, void *ids, void *weights, void *hPairs,
                                    cudaStream_t stream) {
    Engine &e = *(Engine *)h;
    const dl::EngineConfig &c = e.cfg;
    const uint32_t k = c.nActiveExperts;
    if (c.nExperts == 0) return -1;
    if (tensorCores) {
        if (rows > c.maxPrefill) return -1;
        return dl::moePrefillScratchRead(rows, k, c.nExperts, c.ffDim, (float *)logits, (int *)ids, (float *)weights,
                                         (__nv_bfloat16 *)hPairs, stream);
    }
    if (rows != 1) return -1;
    void *dst[4] = {logits, ids, weights, hPairs};
    const void *src[4] = {e.g.routerLogits, e.g.expertIdx, e.g.expertWeight, e.g.h};
    const size_t bytes[4] = {(size_t)c.nExperts * 4, (size_t)k * 4, (size_t)k * 4, (size_t)k * c.ffDim * 4};
    for (int i = 0; i < 4; i++)
        if (dst[i]) DL_CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], bytes[i], cudaMemcpyDeviceToDevice, stream));
    return 0;
}

DL_EXPORT int dl_engine_set_prefill_min_tc(void *h, uint32_t n) { ((Engine *)h)->prefillMinTc = n; return 0; }

// Captures one greedy decode step (forward of 1 token + argmax + position advance) into a graph, after a warm-up forward on
// `stream` that sets kernel attributes outside of capture. Without greedyAdvance no kernel writes tokens, pos or history.
static int captureDecode(Engine *e, cudaStream_t stream) {
    DL_TRY(dl::engineForward(*e, 1, 1, false, stream));
    DL_CUDA_CHECK(cudaStreamSynchronize(stream));
    if (!e->captureStream) DL_CUDA_CHECK(cudaStreamCreateWithFlags(&e->captureStream, cudaStreamNonBlocking));
    DL_CUDA_CHECK(cudaStreamBeginCapture(e->captureStream, cudaStreamCaptureModeThreadLocal));
    const int r = dl::engineForward(*e, 1, 1, true, e->captureStream);
    cudaGraph_t graph = nullptr;
    const cudaError_t endErr = cudaStreamEndCapture(e->captureStream, &graph);
    if (r != 0) { if (graph) cudaGraphDestroy(graph); return r; }
    DL_CUDA_CHECK(endErr);
    DL_CUDA_CHECK(cudaGraphInstantiate(&e->decodeGraph, graph, 0));
    cudaGraphDestroy(graph);
    return 0;
}

// Replays the captured step `nSteps` times back to back on `stream` (no host sync in between), capturing it first if the
// engine has no graph of its current configuration.
DL_EXPORT int dl_engine_decode_graph(void *h, int nSteps, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    if (!e->decodeGraph) DL_TRY(captureDecode(e, stream));
    for (int i = 0; i < nSteps; i++) DL_CUDA_CHECK(cudaGraphLaunch(e->decodeGraph, stream));
    return 0;
}

DL_EXPORT int dl_engine_graph_captured(void *h) { return ((Engine *)h)->decodeGraph ? 1 : 0; }

DL_EXPORT void dl_abi_struct_sizes(uint32_t out[4]) {
    out[0] = sizeof(dl::EngineConfig); out[1] = sizeof(dl::LayerPtrs); out[2] = sizeof(dl::GlobalPtrs); out[3] = sizeof(dl::CommPtrs);
}

// ---- KV-cache slots: up to 8 independent sequences decoded together (attn_decode.cu) -------------------------------------------------

// The layout of the next dl_engine_set_slots: 0 = split (every slot owns floor(seqLen / n) contiguous rows), 1 = paged (the slots
// share every layer plane as one pool of floor(seqLen / 64) pages of 64 rows; a slot holds the pages dl_engine_slot_reserve gave it).
// -64 once slots are set.
DL_EXPORT int dl_engine_set_slot_cache(void *h, int paged) {
    Engine *e = (Engine *)h;
    if (e->slots > 1) return -64;
    if (paged && e->cfg.seqLen < dl::kPageRows) return -61;
    // a paged slot's prompt runs on the tensor-core prefill attention only (launchAttnPrefillTc: head dim 64 or 128, <= 128 q-heads per KV head)
    const dl::EngineConfig &c = e->cfg;
    const bool tcShape = (c.headDim == 64 || c.headDim == 128) && c.nKvHeads && c.nHeads % c.nKvHeads == 0 && c.nHeads / c.nKvHeads <= 128;
    if (paged && (!e->tcAttn || !tcShape)) return -69;
    e->pagedSlots = paged != 0;
    return 0;
}

// Splits every layer's K/V cache into n equal slots of floor(seqLen / n) rows (no extra memory) and allocates the per-slot sampling
// state; paged (dl_engine_set_slot_cache): n slots over one pool of pages, every page free. Single GPU, dense (non-MoE) q40 layers
// only. n = 1 leaves the engine exactly as it was.
DL_EXPORT int dl_engine_set_slots(void *h, uint32_t n) {
    Engine *e = (Engine *)h;
    const dl::EngineConfig &c = e->cfg;
    if (n < 1 || n > kChoiceRngSlots) return -61;
    if (n > 1 && (e->comm.nRanks > 1 || c.nExperts > 0 || c.wType != 0)) return -62;
    uint32_t nb = 1;
    while (nb < n) nb *= 2;
    if (nb > c.maxBatch) return -63;
    e->slots = n;
    e->slotLen = e->pagedSlots && n > 1 ? c.seqLen / dl::kPageRows * dl::kPageRows : c.seqLen / n;
    if (n == 1) return 0;
    if (e->pagedSlots) {
        const uint32_t pages = c.seqLen / dl::kPageRows;
        if (!e->pageDev) {
            DL_CUDA_CHECK(cudaMalloc(&e->pageDev, (size_t)kChoiceRngSlots * pages * sizeof(int32_t)));
            DL_CUDA_CHECK(cudaHostAlloc((void **)&e->pageHost, (size_t)kChoiceRngSlots * pages * sizeof(int32_t), cudaHostAllocDefault));
            DL_CUDA_CHECK(cudaEventCreateWithFlags(&e->pagesStaged, cudaEventDisableTiming));
        }
        DL_CUDA_CHECK(cudaEventSynchronize(e->pagesStaged));
        e->nPages = pages;
        std::fill(e->pageHost, e->pageHost + (size_t)kChoiceRngSlots * pages, -1);
        e->slotPages.assign(kChoiceRngSlots, 0);
        e->pageUsed.assign(pages, 0);
        e->pagesDirty = true;
    }
    DL_TRY(ensureSampler(e));
    DL_TRY(ensureCounts(e, 0));
    const uint32_t full = c.vocab;
    if (!e->slotParams) {
        DL_CUDA_CHECK(cudaMalloc(&e->slotParams, kChoiceRngSlots * 4 * sizeof(float)));
        DL_CUDA_CHECK(cudaMemset(e->slotParams, 0, kChoiceRngSlots * 4 * sizeof(float)));
        DL_CUDA_CHECK(cudaMalloc(&e->slotBias, (size_t)kChoiceRngSlots * full * sizeof(float)));
        DL_CUDA_CHECK(cudaMemset(e->slotBias, 0, (size_t)kChoiceRngSlots * full * sizeof(float)));
        DL_CUDA_CHECK(cudaMalloc(&e->slotFiltersDev, kChoiceRngSlots * sizeof(dl::SampleFilters)));
        DL_CUDA_CHECK(cudaMemset(e->slotFiltersDev, 0, kChoiceRngSlots * sizeof(dl::SampleFilters)));
        DL_CUDA_CHECK(cudaHostAlloc((void **)&e->slotStage, 3 * kChoiceRngSlots * sizeof(int32_t), cudaHostAllocDefault));
        DL_CUDA_CHECK(cudaEventCreateWithFlags(&e->slotStaged, cudaEventDisableTiming));
    }
    DL_CUDA_CHECK(cudaDeviceSynchronize());
    return 0;
}

DL_EXPORT uint32_t dl_engine_slot_len(void *h) {
    Engine *e = (Engine *)h;
    return e->slots > 1 ? e->slotLen : e->cfg.seqLen;
}

DL_EXPORT int dl_engine_slot_reserve(void *h, uint32_t slot, uint32_t rows);

// Paged slots: copies rows [0, P) of slot src into the pages of slot dst (reserved first; -68 and nothing copied when the pool is
// short), one copy per run of pages that are consecutive in both slots.
static int slotCopyPaged(Engine *e, uint32_t src, uint32_t dst, uint32_t P, cudaStream_t stream) {
    const dl::EngineConfig &c = e->cfg;
    if ((uint64_t)P > (uint64_t)e->slotPages[src] * dl::kPageRows) return -60;
    DL_TRY(dl_engine_slot_reserve(e, dst, P));
    const int32_t *ts = e->pageHost + (size_t)src * e->nPages, *td = e->pageHost + (size_t)dst * e->nPages;
    const bool q8 = c.kvType != 0;
    const size_t rowBytes[2] = {(size_t)c.headDim * (q8 ? 1 : sizeof(__nv_bfloat16)), (size_t)c.headDim / 16};
    const uint32_t pages = (P + dl::kPageRows - 1) / dl::kPageRows;
    for (uint32_t i = 0; i < pages;) {
        uint32_t n = 1;
        while (i + n < pages && ts[i + n] == ts[i] + (int32_t)n && td[i + n] == td[i] + (int32_t)n) n++;
        const size_t rows = std::min<size_t>((size_t)n * dl::kPageRows, P - (size_t)i * dl::kPageRows);
        for (const dl::LayerPtrs &L : e->layers)
            for (int plane = 0; plane < (q8 ? 2 : 1); plane++) {
                const size_t pitch = (size_t)c.seqLen * rowBytes[plane];
                for (void *cache : {plane ? L.kScale : L.kCache, plane ? L.vScale : L.vCache})
                    DL_CUDA_CHECK(cudaMemcpy2DAsync((uint8_t *)cache + (size_t)td[i] * dl::kPageRows * rowBytes[plane], pitch,
                                                    (const uint8_t *)cache + (size_t)ts[i] * dl::kPageRows * rowBytes[plane], pitch,
                                                    rows * rowBytes[plane], c.nKvHeads, cudaMemcpyDeviceToDevice, stream));
            }
        i += n;
    }
    return 0;
}

// Copies rows [0, P) of slot src into slot dst, every layer and KV head (several completions of one prompt). Paged slots: into
// dst's own pages, reserved first (-68 when the pool is short).
DL_EXPORT int dl_engine_slot_copy(void *h, uint32_t src, uint32_t dst, uint32_t P, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    const dl::EngineConfig &c = e->cfg;
    if (e->slots < 2 || src >= e->slots || dst >= e->slots || P > e->slotLen) return -64;
    if (src == dst || P == 0) return 0;
    if (e->pagedSlots) return slotCopyPaged(e, src, dst, P, stream);
    // bf16: one plane per cache; q80: the int8 values (headDim bytes a row) and the scales (headDim / 16 bytes a row)
    const bool q8 = c.kvType != 0;
    const size_t rowBytes[2] = {(size_t)c.headDim * (q8 ? 1 : sizeof(__nv_bfloat16)), (size_t)c.headDim / 16};
    for (const dl::LayerPtrs &L : e->layers)
        for (int plane = 0; plane < (q8 ? 2 : 1); plane++) {
            const size_t pitch = (size_t)e->slotLen * rowBytes[plane], slotBytes = (size_t)c.nKvHeads * pitch;
            for (void *cache : {plane ? L.kScale : L.kCache, plane ? L.vScale : L.vCache})
                DL_CUDA_CHECK(cudaMemcpy2DAsync((uint8_t *)cache + dst * slotBytes, pitch, (const uint8_t *)cache + src * slotBytes, pitch,
                                                (size_t)P * rowBytes[plane], c.nKvHeads, cudaMemcpyDeviceToDevice, stream));
        }
    return 0;
}

// The sampling settings of the sequence admitted to slot `slot`: seeds its generator (rngState[kChoiceRngSlots + slot]), zeroes its
// count row (1 + slot) and sets its temperature (0: arg-max), top-p, penalties and logit bias (nBias (id, value) pairs, ids below the
// sampled vocabulary). The uploads are complete when the call returns.
DL_EXPORT int dl_engine_slot_sampling(void *h, uint32_t slot, unsigned long long seed, float temperature, float topp, float presence,
                                      float frequency, const int32_t *ids, const float *vals, int nBias, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    if (e->slots < 2 || slot >= e->slots) return -64;
    const uint32_t full = e->cfg.vocab;
    const uint32_t n = (e->vocabLimit && e->vocabLimit < full) ? e->vocabLimit : full;
    if (!(temperature >= 0.f) || nBias < 0) return -52;
    for (int i = 0; i < nBias; i++) if (ids[i] < 0 || (uint32_t)ids[i] >= n) return -53;
    if (seed == 0) seed = 0x9E3779B97F4A7C15ull;   // xorshift state must not be zero
    std::vector<float> bias(full, 0.f);
    for (int i = 0; i < nBias; i++) bias[ids[i]] = vals[i];
    const float params[4] = {temperature, topp, presence, frequency};
    DL_CUDA_CHECK(cudaMemcpyAsync(e->rngState + kChoiceRngSlots + slot, &seed, sizeof(seed), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(e->slotParams + 4 * slot, params, sizeof(params), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(e->slotBias + (size_t)slot * full, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaMemsetAsync(e->ctlCounts + (size_t)(1 + slot) * full, 0, (size_t)full * sizeof(uint32_t), stream));
    if (filtersOn(e->slotFilters[slot])) {   // a new sequence starts without filters (dl_engine_slot_filters)
        e->slotFilters[slot] = dl::SampleFilters{};
        DL_CUDA_CHECK(cudaMemsetAsync(e->slotFiltersDev + slot, 0, sizeof(dl::SampleFilters), stream));
    }
    DL_CUDA_CHECK(cudaStreamSynchronize(stream));   // host temporaries
    e->slotLogprobs[slot] = -1;   // a new sequence starts without logprobs (dl_engine_slot_logprobs)
    return 0;
}

// top_k / min_p (kernels.h: SampleFilters) of slot `slot`'s sampled draws, for the sequence admitted by the last
// dl_engine_slot_sampling (which switches them off). The upload is complete when the call returns.
DL_EXPORT int dl_engine_slot_filters(void *h, uint32_t slot, uint32_t topK, float minP) {
    Engine *e = (Engine *)h;
    if (e->slots < 2 || slot >= e->slots) return -64;
    const dl::SampleFilters f{topK, minP};
    if (!dl::sampleFiltersValid(f)) return -54;
    DL_CUDA_CHECK(cudaMemcpy(e->slotFiltersDev + slot, &f, sizeof(f), cudaMemcpyHostToDevice));
    e->slotFilters[slot] = f;
    return 0;
}

// Rows of a slots step: the power of two >= slots, so a row's arithmetic does not depend on how many slots are busy.
static int slotRows(const Engine *e) {
    int nb = 1;
    while ((uint32_t)nb < e->slots) nb *= 2;
    return nb;
}

// Forward of one slots step: row b feeds tokens[b] at position pos[b] (host arrays of `slots` entries) and writes K/V row pos[b]
// of slot b. Rows set in inactiveMask (and the padding rows up to the power of two) write nothing. Logits of every row land in
// logits[0..nb).
DL_EXPORT int dl_engine_slots_forward(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, cudaStream_t stream) {
    Engine *e = (Engine *)h;
    if (e->slots < 2) return -64;
    const int nb = slotRows(e);
    uint32_t mask = inactiveMask;
    for (int b = (int)e->slots; b < nb; b++) mask |= 1u << b;
    if ((mask & ((1u << nb) - 1u)) == ((1u << nb) - 1u)) return -65;   // nothing to run
    int32_t *tok = e->slotStage, *ps = e->slotStage + kChoiceRngSlots;
    DL_CUDA_CHECK(cudaEventSynchronize(e->slotStaged));   // the previous call's uploads have read the staging buffer
    for (int b = 0; b < nb; b++) {
        const bool on = !((mask >> b) & 1u);
        if (on && (pos[b] < 0 || (uint32_t)pos[b] >= e->slotLen)) return -66;
        if (on && e->pagedSlots && (uint32_t)pos[b] >= e->slotPages[b] * dl::kPageRows) return -66;   // not reserved
        tok[b] = on ? tokens[b] : 0;
        ps[b] = on ? pos[b] : 0;
    }
    DL_CUDA_CHECK(cudaMemcpyAsync(e->g.tokens, tok, nb * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(e->g.pos, ps, nb * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaEventRecord(e->slotStaged, stream));
    if (e->pagedSlots) DL_TRY(uploadPages(e, stream));
    const dl::SlotStep sl{mask};
    return dl::engineForward(*e, nb, 2, false, stream, nullptr, &sl);
}

// Log-probabilities of slot `slot`'s draws in dl_engine_slots_step_logprobs: k (0..20) top entries, -1: none (the default).
DL_EXPORT int dl_engine_slot_logprobs(void *h, uint32_t slot, int k) {
    Engine *e = (Engine *)h;
    if (e->slots < 2 || slot >= e->slots) return -64;
    if (k < -1 || k > dl::kLogprobsMaxTop) return -67;
    e->slotLogprobs[slot] = k;
    return 0;
}

// dl_engine_slots_forward, then every active row draws its next token with its slot's settings (dl_engine_slot_sampling) into
// out[b]; inactive rows leave out[b] as it was. One device-to-host copy for all rows; returns once the tokens are on the host.
// lpOut (host int32 [slots][kLogprobsWords], may be null): an active row whose slot has logprobs on (dl_engine_slot_logprobs) also
// gets the log-probabilities of its draw there (kernels.h: launchLogprobsRows), computed behind the draw and copied out with the
// tokens; other rows of lpOut are left as they were, and without such a row nothing more runs.
DL_EXPORT int dl_engine_slots_step_logprobs(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, int32_t *out, int32_t *lpOut,
                                            cudaStream_t stream) {
    Engine *e = (Engine *)h;
    DL_TRY(dl_engine_slots_forward(h, tokens, pos, inactiveMask, stream));
    const dl::EngineConfig &c = e->cfg;
    const int nb = slotRows(e);
    uint32_t mask = inactiveMask;
    for (int b = (int)e->slots; b < nb; b++) mask |= 1u << b;
    const uint32_t n = (e->vocabLimit && e->vocabLimit < c.vocab) ? e->vocabLimit : c.vocab;
    const dl::SampleControls ctl{e->slotBias, e->ctlCounts + c.vocab, c.vocab, 0.f, 0.f, c.vocab};
    bool anyFilters = false;
    for (uint32_t b = 0; b < e->slots; b++) anyFilters = anyFilters || (!((mask >> b) & 1u) && filtersOn(e->slotFilters[b]));
    DL_TRY(dl::launchSampleRows(e->g.logits, c.vocab, e->probScratch, n, 0.f, 0.f, e->rngState + kChoiceRngSlots, e->g.tokens, (uint32_t)nb, mask,
                                nullptr, nullptr, 1, stream, &ctl, e->slotParams, nullptr, anyFilters ? e->slotFiltersDev : nullptr));
    uint32_t lpMask = 0;
    int lpK[kChoiceRngSlots] = {};
    for (uint32_t b = 0; lpOut && b < e->slots; b++)
        if (!((mask >> b) & 1u) && e->slotLogprobs[b] >= 0) { lpMask |= 1u << b; lpK[b] = e->slotLogprobs[b]; }
    if (lpMask) {
        if (!e->slotLpDev) {
            DL_CUDA_CHECK(cudaMalloc(&e->slotLpDev, kChoiceRngSlots * dl::kLogprobsWords * sizeof(int32_t)));
            DL_CUDA_CHECK(cudaHostAlloc((void **)&e->slotLpHost, kChoiceRngSlots * dl::kLogprobsWords * sizeof(int32_t), cudaHostAllocDefault));
        }
        DL_TRY(dl::launchLogprobsRows(e->g.logits, c.vocab, n, (uint32_t)nb, lpMask, lpK, e->g.tokens, e->slotLpDev, stream, &ctl, e->slotParams));
        DL_CUDA_CHECK(cudaMemcpyAsync(e->slotLpHost, e->slotLpDev, (size_t)nb * dl::kLogprobsWords * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    }
    int32_t *drawn = e->slotStage + 2 * kChoiceRngSlots;
    DL_CUDA_CHECK(cudaMemcpyAsync(drawn, e->g.tokens, nb * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    DL_CUDA_CHECK(cudaStreamSynchronize(stream));
    for (uint32_t b = 0; b < e->slots; b++) if (!((mask >> b) & 1u)) out[b] = drawn[b];
    for (uint32_t b = 0; b < e->slots; b++)
        if ((lpMask >> b) & 1u) std::memcpy(lpOut + b * dl::kLogprobsWords, e->slotLpHost + b * dl::kLogprobsWords, dl::kLogprobsWords * sizeof(int32_t));
    return 0;
}

DL_EXPORT int dl_engine_slots_step(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, int32_t *out, cudaStream_t stream) {
    return dl_engine_slots_step_logprobs(h, tokens, pos, inactiveMask, out, nullptr, stream);
}

// ---- paged slots: the page allocator (dl_engine_set_slot_cache) -------------------------------------------------------------------

// Grows slot `slot`'s pages to cover rows [0, rows), free pages taken lowest index first. -68 when the pool has too few free pages
// (nothing changes then); -60 past the slot length.
DL_EXPORT int dl_engine_slot_reserve(void *h, uint32_t slot, uint32_t rows) {
    Engine *e = (Engine *)h;
    if (!e->pagedSlots || e->slots < 2 || slot >= e->slots) return -64;
    if (rows > e->slotLen) return -60;
    const uint32_t need = (rows + dl::kPageRows - 1) / dl::kPageRows;
    uint32_t &have = e->slotPages[slot];
    if (need <= have) return 0;
    if ((uint32_t)std::count(e->pageUsed.begin(), e->pageUsed.end(), 0) < need - have) return -68;
    DL_TRY(editPages(e));
    int32_t *row = e->pageHost + (size_t)slot * e->nPages;
    for (uint32_t p = 0; p < e->nPages && have < need; p++)
        if (!e->pageUsed[p]) { e->pageUsed[p] = 1; row[have++] = (int32_t)p; }
    return 0;
}

// Returns every page of slot `slot` to the pool.
DL_EXPORT int dl_engine_slot_release(void *h, uint32_t slot) {
    Engine *e = (Engine *)h;
    if (!e->pagedSlots || e->slots < 2 || slot >= e->slots) return -64;
    if (e->slotPages[slot] == 0) return 0;
    DL_TRY(editPages(e));
    int32_t *row = e->pageHost + (size_t)slot * e->nPages;
    for (uint32_t i = 0; i < e->slotPages[slot]; i++) { e->pageUsed[row[i]] = 0; row[i] = -1; }
    e->slotPages[slot] = 0;
    return 0;
}

// Shrinks slot `slot` to the pages that cover rows [0, rows) and returns the rest to the pool (a slot taken by a request that needs
// fewer rows than its previous occupant left).
DL_EXPORT int dl_engine_slot_trim(void *h, uint32_t slot, uint32_t rows) {
    Engine *e = (Engine *)h;
    if (!e->pagedSlots || e->slots < 2 || slot >= e->slots) return -64;
    const uint32_t keep = (rows + dl::kPageRows - 1) / dl::kPageRows;
    if (keep >= e->slotPages[slot]) return 0;
    DL_TRY(editPages(e));
    int32_t *row = e->pageHost + (size_t)slot * e->nPages;
    for (uint32_t i = keep; i < e->slotPages[slot]; i++) { e->pageUsed[row[i]] = 0; row[i] = -1; }
    e->slotPages[slot] = keep;
    return 0;
}

// Free pages of the pool (0 without paged slots).
DL_EXPORT uint32_t dl_engine_free_pages(void *h) {
    Engine *e = (Engine *)h;
    if (!e->pagedSlots || e->slots < 2) return 0;
    return (uint32_t)std::count(e->pageUsed.begin(), e->pageUsed.end(), 0);
}

// Slot `slot`'s physical pages in logical order into out[0..cap); returns how many it holds (negative: not paged).
DL_EXPORT int dl_engine_slot_pages(void *h, uint32_t slot, int32_t *out, uint32_t cap) {
    Engine *e = (Engine *)h;
    if (!e->pagedSlots || e->slots < 2 || slot >= e->slots) return -64;
    for (uint32_t i = 0; i < e->slotPages[slot] && i < cap; i++) out[i] = e->pageHost[(size_t)slot * e->nPages + i];
    return (int)e->slotPages[slot];
}

// ---- speculative decoding with a draft model (speculative.cu) ------------------------------------------------------------------------

static int ensureSpec(Engine *e) {
    if (e->spec) return 0;
    dl::Spec *s = new dl::Spec();
    const size_t words = 8 * 256;
    const size_t bytes = words * 4 * 2 + 64 + 32 + dl::kSpecResultWords * 4;
    if (cudaMalloc(&s->dev, bytes) != cudaSuccess || cudaMemset(s->dev, 0, bytes) != cudaSuccess ||
        cudaHostAlloc((void **)&s->stage, (dl::kSpecResultHead + dl::kSpecResultWords) * 4, cudaHostAllocDefault) != cudaSuccess) {
        if (s->dev) cudaFree(s->dev);
        delete s;
        return -77;   // out of device or pinned memory; nothing is kept, a later call tries again
    }
    s->argVal = (float *)s->dev;
    s->argIdx = (int *)(s->dev + words * 4);
    s->argCounter = (unsigned int *)(s->dev + words * 8);
    s->verifyTok = (int *)(s->dev + words * 8 + 64);
    s->result = (int *)(s->dev + words * 8 + 96);
    e->spec = s;
    return 0;
}

// Whether `draft` can draft for `target`: two engines on one rank, dense q40 layers, the same vocabulary and KV-cache storage, no slots.
static int specCheck(const Engine &t, const Engine &d) {
    if (&t == &d) return -72;
    for (const Engine *e : {&t, &d})
        if (e->comm.nRanks > 1 || e->cfg.nExperts > 0 || e->cfg.wType != 0 || e->slots > 1) return -73;
    if (t.cfg.vocab != d.cfg.vocab || t.g.vocabFull != d.g.vocabFull || t.cfg.kvType != d.cfg.kvType) return -72;
    return 0;
}

static dl::SpecAcceptArgs specArgs(Engine &t, Engine &d, uint32_t k) {
    dl::SpecAcceptArgs a{};
    a.verifyTokens = t.spec->verifyTok; a.targetTokens = t.g.tokens; a.targetPos = t.g.pos; a.targetHistory = t.g.history;
    a.historyCap = t.cfg.seqLen; a.draftTokens = d.g.tokens; a.draftPos = d.g.pos; a.draftHistory = d.g.history;
    a.draftHistoryCap = d.cfg.seqLen; a.k = k; a.result = t.spec->result;
    return a;
}

// The launches of one round of k drafts. The draft feeds t, d1..dk (k + 1 greedy steps, the last output unused): so it holds the
// row of dk when every draft is accepted. The target verifies [t, d1..dk] at p..p+k, the accept kernel keeps g(0..a).
static int specRoundLaunches(Engine &t, Engine &d, uint32_t k, cudaStream_t stream) {
    const dl::SpecAcceptArgs a = specArgs(t, d, k);
    DL_TRY(dl::launchSpecStage(a, stream));
    for (uint32_t i = 1; i <= k + 1; i++) {
        DL_TRY(dl::engineForward(d, 1, 1, true, stream));
        if (i <= k) DL_CUDA_CHECK(cudaMemcpyAsync(t.g.tokens + i, d.g.tokens, 4, cudaMemcpyDeviceToDevice, stream));
    }
    DL_TRY(dl::engineForward(t, (int)k + 1, 3, false, stream));
    return dl::launchSpecAccept(a, stream);
}

static int captureSpecRound(Engine &t, Engine &d, uint32_t k) {
    dl::Spec &s = *t.spec;
    if (s.graph[k]) { cudaGraphExecDestroy(s.graph[k]); s.graph[k] = nullptr; }
    if (!t.captureStream) DL_CUDA_CHECK(cudaStreamCreateWithFlags(&t.captureStream, cudaStreamNonBlocking));
    DL_CUDA_CHECK(cudaStreamBeginCapture(t.captureStream, cudaStreamCaptureModeThreadLocal));
    const int r = specRoundLaunches(t, d, k, t.captureStream);
    cudaGraph_t graph = nullptr;
    const cudaError_t endErr = cudaStreamEndCapture(t.captureStream, &graph);
    if (r != 0) { if (graph) cudaGraphDestroy(graph); return r; }
    DL_CUDA_CHECK(endErr);
    DL_CUDA_CHECK(cudaGraphInstantiate(&s.graph[k], graph, 0));
    cudaGraphDestroy(graph);
    s.graphDraft[k] = d.serial;
    s.graphGen[k][0] = t.graphGen;
    s.graphGen[k][1] = d.graphGen;
    return 0;
}

// One round of speculative decoding: the last emitted token `token` sits at position `pos`, and both engines hold valid KV rows for
// every position before it. k (1, 3 or 7) drafts, fewer where pos + k would reach the end of either cache; at the last row one
// greedy step of each engine (k = 0). Writes the result block (kSpecResultWords int32, layout in kernels.h) to `out` once the
// round has finished on `stream`. useGraph: replay the round's graph (captured after the first eager round of each k).
DL_EXPORT int dl_spec_round(void *target, void *draft, int token, int pos, int k, int useGraph, int32_t *out, cudaStream_t stream) {
    Engine &t = *(Engine *)target, &d = *(Engine *)draft;
    DL_TRY(specCheck(t, d));
    if (k != 1 && k != 3 && k != 7) return -75;
    const uint32_t seqLen = std::min(t.cfg.seqLen, d.cfg.seqLen);
    if (pos < 0 || (uint32_t)pos >= seqLen) return -71;
    while (k > 0 && (uint32_t)(pos + k) >= seqLen) k /= 2;   // 7 -> 3 -> 1 -> 0
    if ((uint32_t)k + 1 > t.cfg.maxBatch) return -10;
    DL_TRY(ensureSpec(&t));
    dl::Spec &s = *t.spec;
    int32_t *res = s.stage + dl::kSpecResultHead;
    s.stage[0] = token;
    s.stage[1] = pos;
    DL_CUDA_CHECK(cudaMemcpyAsync(t.g.tokens, s.stage, 4, cudaMemcpyHostToDevice, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(t.g.pos, s.stage + 1, 4, cudaMemcpyHostToDevice, stream));
    if (k == 0) {
        DL_CUDA_CHECK(cudaMemcpyAsync(d.g.tokens, s.stage, 4, cudaMemcpyHostToDevice, stream));
        DL_CUDA_CHECK(cudaMemcpyAsync(d.g.pos, s.stage + 1, 4, cudaMemcpyHostToDevice, stream));
        for (Engine *e : {&t, &d}) {
            if (useGraph) DL_TRY(dl_engine_decode_graph(e, 1, stream));
            else DL_TRY(dl::engineForward(*e, 1, 1, true, stream));
        }
        DL_CUDA_CHECK(cudaMemcpyAsync(res + dl::kSpecResultHead, t.g.tokens, 4, cudaMemcpyDeviceToHost, stream));
        DL_CUDA_CHECK(cudaStreamSynchronize(stream));
        res[0] = 0; res[1] = 1; res[2] = 0; res[3] = pos + 1;
    } else {
        const bool fresh = s.graph[k] && s.graphDraft[k] == d.serial && s.graphGen[k][0] == t.graphGen && s.graphGen[k][1] == d.graphGen;
        if (useGraph && fresh) DL_CUDA_CHECK(cudaGraphLaunch(s.graph[k], stream));
        else DL_TRY(specRoundLaunches(t, d, (uint32_t)k, stream));   // the first round of a k also sets the kernels' attributes
        DL_CUDA_CHECK(cudaMemcpyAsync(res, s.result, dl::kSpecResultWords * 4, cudaMemcpyDeviceToHost, stream));
        DL_CUDA_CHECK(cudaStreamSynchronize(stream));
        if (useGraph && !fresh) DL_TRY(captureSpecRound(t, d, (uint32_t)k));
    }
    if (dl_engine_aborted(&t) || dl_engine_aborted(&d)) return -74;
    std::memcpy(out, res, dl::kSpecResultWords * 4);
    return 0;
}

// The verify step alone (tests): nb (2, 4 or 8) tokens staged in tokens[0..nb) at pos[0..nb), logits of every row into logits[0..nb)
// and the arg-max of row b (ids >= the vocabulary limit ignored, lowest id among ties) into out[b] once the stream has finished.
DL_EXPORT int dl_engine_verify(void *h, int nb, int32_t *out, cudaStream_t stream) {
    Engine &e = *(Engine *)h;
    DL_TRY(ensureSpec(&e));
    DL_TRY(dl::engineForward(e, nb, 3, false, stream));
    DL_CUDA_CHECK(cudaMemcpyAsync(e.spec->stage, e.spec->verifyTok, nb * 4, cudaMemcpyDeviceToHost, stream));
    DL_CUDA_CHECK(cudaStreamSynchronize(stream));
    std::memcpy(out, e.spec->stage, nb * 4);
    return 0;
}

DL_EXPORT uint32_t dl_spec_result_words() { return dl::kSpecResultWords; }
