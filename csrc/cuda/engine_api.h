// C ABI of the per-rank engine in _cuda.so: plain structs + extern "C" entry points. Shared by engine.cu, the ctypes mirror in
// distributed_llama_b200/ops/cuda_lib.py and the native (Python-free) runtime under csrc/app/.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace dl {

constexpr int kApiMaxRanks = 8;
constexpr int kApiLogprobsWords = 44;   // int32 words of one row's log-probabilities (dl_engine_logprobs)
constexpr int kApiLogprobsMaxTop = 20;
constexpr int kLogprobsControlled = 1, kLogprobsSharedRow = 2;   // dl_engine_logprobs flags
constexpr int kEngineErrPoolShort = -68;   // dl_engine_slot_reserve / dl_engine_slot_copy: too few free pages, nothing changed

struct EngineConfig {   // mirrored by ctypes in distributed_llama_b200/ops/cuda_lib.py
    uint32_t dim, nLayers, nHeads, nKvHeads, headDim, ffDim, vocab, seqLen;   // per-rank (sliced) head/ff/vocab counts
    uint32_t nExperts, nActiveExperts;
    uint32_t maxBatch;       // tokens per forward on the GEMV path
    uint32_t nSplits;        // attention KV splits
    uint32_t rank, nRanks;
    uint32_t numSms;
    float eps;
    uint32_t usePdl;
    uint32_t moeFirstExpert, moeNumLocal;   // experts held by this rank (expert parallelism); TP mode: 0, nExperts
    uint32_t wType;          // matrix storage: 0 = q40 device layout, 1 = dense f32, 2 = dense f16 (gemv_dense.cu)
    uint32_t hiddenAct;      // gate activation: 0 = SiLU, 1 = GELU (tanh form) — the `.m` header's hidden_act
    uint32_t kvType;         // KV-cache storage: 0 = bf16, 1 = q80 (int8 values + f16 scale per 32, LayerPtrs::kScale / vScale)
    uint32_t maxPrefill;     // tokens per tensor-core prompt chunk, 1..256
};

struct LayerPtrs {
    const void *qkvQs, *qkvSc;   // [(nHeads+2nKvHeads)*hd][dim]
    const void *woQs, *woSc;     // [dim][nHeads*hd]
    const void *w13Qs, *w13Sc;   // [2*ff][dim] (gate/up interleaved); MoE: [nExperts][2*ff][dim]
    const void *w2Qs, *w2Sc;     // [dim][ff];                          MoE: [nExperts][dim][ff]
    const float *norm0, *norm1, *qNorm, *kNorm;
    const float *moeGate;        // [nExperts][dim] f32
    void *kCache, *vCache;       // bf16 [nKvHeads][seqLen][hd]; kvType 1: int8 [nKvHeads][seqLen][hd]
    void *kScale, *vScale;       // kvType 1: f16 [nKvHeads][seqLen][hd / 32] + 16 bytes of tail padding; unused for bf16
};

struct GlobalPtrs {   // the engine allocates its scratch buffers itself (dl_engine_create)
    const float *embedding;      // [vocabFull][dim] (replicated) or this rank's shard when embRowsPerRank != 0
    const float *embeddingPeers[kApiMaxRanks];   // vocabulary shards of all ranks (peer-mapped), used when embRowsPerRank != 0
    uint32_t embRowsPerRank;     // 0: `embedding` is the whole table
    const float *finalNorm;
    const void *wclsQs, *wclsSc; // [vocab][dim]
    const float *rope;           // [seqLen][hd/2][2]
    uint32_t vocabFull;
    // buffers the client reads or writes
    int *tokens, *pos;           // [maxBatch]
    float *x;                    // [maxBatch][dim] residual stream (the library-collective path adds its all-reduced partials here)
    float *logits;               // [maxBatch][vocab]
    int *history;                // [seqLen] generated token per position (device-side log), may be null
};

struct CommPtrs {   // mirrored by ctypes; the engine lays out the arena itself (dl_engine_arena_bytes)
    uint32_t nRanks, rank;
    void *arena[kApiMaxRanks];          // every rank's symmetric arena mapped into this process
    void *mcArena;                      // NVLS multicast mapping of the arena (null: none)
};

}  // namespace dl

extern "C" {
void *dl_engine_create(const dl::EngineConfig *cfg);   // null on an unsupported configuration or a failed allocation
void dl_engine_destroy(void *h);
int dl_engine_set_layer(void *h, uint32_t layer, const dl::LayerPtrs *p);
int dl_engine_set_globals(void *h, const dl::GlobalPtrs *p);
uint64_t dl_engine_arena_bytes(void *h);   // size of the symmetric peer-memory arena, after dl_engine_set_globals
int dl_engine_set_comm(void *h, const dl::CommPtrs *p);
int dl_engine_enable_mega(void *h, int enable);
int dl_engine_set_vocab_limit(void *h, uint32_t limit);   // greedy arg-max never returns ids >= limit (tokenizer vocabulary size)
int dl_engine_aborted(void *h);
int dl_engine_mega_active(void *h);   // 1 if the last single-token forward ran on the persistent kernel (0: fell back to the multi-kernel path)
// Copies the persistent kernel's x, q|k|v, z (LL words) and SwiGLU (f32) vectors with their 8 tail words into device memory (tests).
int dl_engine_mega_copy_vectors(void *h, void *x, void *qkv, void *z, void *hF, cudaStream_t stream);
unsigned long long dl_engine_sync_ns(void *h);
int dl_engine_sampler_seed(void *h, unsigned long long seed);
int dl_engine_sample(void *h, float temperature, float topp, cudaStream_t stream);   // after a forward with logitsMode 1
// presence / frequency penalties and logit bias of the following draws; zeroes the count rows in rowMask (bit 0: single sequence,
// bit 1 + b: choice b). All zero: off.
int dl_engine_set_sampling_controls(void *h, float presence, float frequency, const int32_t *ids, const float *vals, int nBias, uint32_t rowMask,
                                    cudaStream_t stream);
// top_k / min_p of the following sampled draws of the single sequence and the choices (kernels.h: SampleFilters); 0 / 0: off.
// minP in [0, 1]. They persist until changed.
int dl_engine_set_sampling_filters(void *h, uint32_t topK, float minP);
// choices (several completions of one prompt, csrc/cuda/attn_decode.cu): generators 0..n-1, batched draws, one choices forward
int dl_engine_sampler_seed_rows(void *h, const unsigned long long *seeds, int n);   // separate from the single-sequence generator
unsigned long long dl_engine_sampler_state(void *h);   // single-sequence generator state (seed with it to continue the stream)
int dl_engine_sample_rows(void *h, int nb, uint32_t inactiveMask, float temperature, float topp, int firstStep, cudaStream_t stream);
int dl_engine_choices_forward(void *h, int nb, uint32_t P, uint32_t C, uint32_t j, uint32_t inactiveMask, cudaStream_t stream);
// KV-cache slots (csrc/cuda/attn_decode.cu): n <= 8 independent sequences, slot s = rows [0, floor(seqLen / n)) of its own cache block
int dl_engine_set_slots(void *h, uint32_t n);
uint32_t dl_engine_slot_len(void *h);
// Paged slots: set paged = 1 before dl_engine_set_slots and the slots share every layer plane as one pool of floor(seqLen / 64)
// 64-row pages; dl_engine_slot_len is then 64 * floor(seqLen / 64). A slot's rows must be reserved before a step or prefill writes
// them. dl_engine_slot_reserve returns kEngineErrPoolShort, changing nothing, when the pool has too few free pages; pages are taken
// lowest index first.
int dl_engine_set_slot_cache(void *h, int paged);
int dl_engine_slot_reserve(void *h, uint32_t slot, uint32_t rows);
int dl_engine_slot_release(void *h, uint32_t slot);
int dl_engine_slot_trim(void *h, uint32_t slot, uint32_t rows);   // keeps the pages of rows [0, rows), frees the rest
uint32_t dl_engine_free_pages(void *h);
int dl_engine_slot_pages(void *h, uint32_t slot, int32_t *out, uint32_t cap);
int dl_engine_slot_copy(void *h, uint32_t src, uint32_t dst, uint32_t P, cudaStream_t stream);
int dl_engine_slot_sampling(void *h, uint32_t slot, unsigned long long seed, float temperature, float topp, float presence, float frequency,
                            const int32_t *ids, const float *vals, int nBias, cudaStream_t stream);
int dl_engine_slot_filters(void *h, uint32_t slot, uint32_t topK, float minP);   // off after every dl_engine_slot_sampling
int dl_engine_slots_forward(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, cudaStream_t stream);
int dl_engine_slots_step(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, int32_t *out, cudaStream_t stream);
// per-token log-probabilities (csrc/cuda/logprobs.cu): results are int32 blocks of kLogprobsWords words per row,
// {chosen id, its logprob (f32 bits), k, 0, k x (id, logprob bits)} in the order (logprob desc, id asc); flags: bit 0 = the
// sampling controls of the last draw apply, bit 1 = every row reads logits row 0 (the choices' first draw)
int dl_engine_logprobs(void *h, int rows, uint32_t rowMask, const int32_t *k, int firstRow, int flags, int32_t *out, cudaStream_t stream);
int dl_engine_slot_logprobs(void *h, uint32_t slot, int k);
// the kernel on explicit device buffers (csrc/cuda/logprobs.cu: counts are those after the draws of chosen[b])
int dl_logprobs_rows(const float *logits, uint32_t logitsStride, uint32_t n, uint32_t B, uint32_t rowMask, const int *k, const int *chosen,
                     const float *bias, uint32_t biasStride, uint32_t *counts, uint32_t countsStride, float presence, float frequency,
                     const float *rowParams, int32_t *out, cudaStream_t stream);   // k = -1: off (every dl_engine_slot_sampling resets it)
int dl_engine_slots_step_logprobs(void *h, const int32_t *tokens, const int32_t *pos, uint32_t inactiveMask, int32_t *out, int32_t *lpOut,
                                  cudaStream_t stream);
int dl_engine_set_trace(void *h, uint64_t *buf, uint32_t capLaunches);
int dl_engine_set_trace_all(void *h, int allCtas);
uint32_t dl_engine_num_sms(void *h);
int dl_engine_forward(void *h, int nb, int logitsMode, int greedyAdvance, cudaStream_t stream);
int dl_engine_forward_part(void *h, int nb, uint32_t layer, int part, float *ybuf, cudaStream_t stream);
// n prompt tokens (host memory) at positions p0 .. p0 + n - 1; slot >= 0: into KV-cache slot `slot`
int dl_engine_prefill(void *h, const int32_t *hostTokens, uint32_t n, uint32_t p0, int slot, int wantLogits, cudaStream_t stream);
// the chunks dl_engine_prefill runs, as up to `cap` (T, p0, on tensor cores) triples; returns their number or a negative error
int dl_engine_prefill_plan(void *h, uint32_t n, uint32_t p0, int slot, uint32_t *out, uint32_t cap);
int dl_prefill_plan(uint32_t n, uint32_t p0, int slot, uint32_t slots, uint32_t rows, uint32_t maxPrefill, uint32_t maxBatch,
                    uint32_t minTc, int tcAllowed, uint32_t *out, uint32_t cap);   // the same schedule, no engine or device
// copies the last prompt chunk's scratch intermediates into device memory (tests); null destinations are skipped
int dl_engine_prefill_scratch(void *h, uint32_t rows, void *px, void *pqkv, void *pxn, void *pzb, void *phb, void *qkv, void *z,
                              void *hF, cudaStream_t stream);
int dl_engine_set_prefill_min_tc(void *h, uint32_t n);   // shortest chunk on the tensor cores (default 9; 0: never)
int dl_engine_decode_graph(void *h, int nSteps, cudaStream_t stream);   // captures the greedy step on first use
int dl_engine_graph_captured(void *h);
// one round of greedy speculative decoding with `draft` (engine.cu): result block of dl_spec_result_words() int32 into `out`
int dl_spec_round(void *target, void *draft, int token, int pos, int k, int useGraph, int32_t *out, cudaStream_t stream);
uint32_t dl_spec_result_words();
void dl_abi_struct_sizes(uint32_t out[4]);   // sizeof EngineConfig, LayerPtrs, GlobalPtrs, CommPtrs
// symmetric peer-memory arena (csrc/cuda/comm_vmm.cu): create (local, binds the bootstrap socket) -> [job-wide barrier] -> connect
// (collective: exchanges file descriptors, maps every peer, sets up the NVSwitch multicast mapping)
void *dl_vmm_create(uint32_t rank, uint32_t nRanks, size_t bytes, const char *tag, int wantMulticast);
int dl_vmm_connect(void *h);
void *dl_vmm_ptr(void *h, uint32_t rank);
void *dl_vmm_mc_ptr(void *h);
int dl_vmm_barrier(void *h, uint32_t phase);   // host barrier over the bootstrap sockets, phase 3..14
void dl_vmm_destroy(void *h);
int dl_repack_q40(const void *src, uint64_t srcRowPitch, uint64_t srcColByteOffset, uint32_t rows, uint32_t blocksPerRow, void *dstQs,
                  void *dstScales, uint32_t dstRowStride, uint32_t dstRowOffset, uint32_t headDim, cudaStream_t stream);
}
