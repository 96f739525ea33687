// Python-free runtime of one GPU: maps a `.m` file, uploads + re-tiles the q40 weights, owns the device buffers and drives the
// engine in _cuda.so (persistent decode kernel, tensor-core prefill, CUDA-graph greedy loop).
//
// Role in the reference: loadLlmNetWeight + NnExecutor/NnCpuDevice set-up + RootLlmInference (src/llm.cpp:614-669,
// src/nn/nn-cpu.cpp:41-148, src/app.cpp:168-208) for the single-node case. The tensor-parallel launcher (one process per GPU,
// torch.distributed bootstrap, peer-memory arena) lives in the Python package; this class is what `dllama-native` and embedders
// that do not want an interpreter link against.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <utility>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../host/model_format.hpp"

namespace dl {

// --kv-cache-float-type {bf16|q80} -> EngineConfig::kvType; throws std::runtime_error on anything else.
inline uint32_t parseKvCacheFloatType(const std::string &v) {
    if (v == "bf16") return 0;
    if (v == "q80") return 1;
    throw std::runtime_error("Invalid KV-cache float type: " + v + " (expected bf16 or q80)");
}

// Device bytes of one rank's K and V caches: bf16 = 2 bytes a value, q80 = 1 byte a value + a 2-byte scale per 32.
inline uint64_t kvCacheBytes(const ModelHeader &h, uint32_t nRanks, uint32_t kvType) {
    const uint64_t kvHeads = h.nKvHeads >= nRanks ? h.nKvHeads / nRanks : 1;
    const uint64_t values = 2ull * h.nLayers * h.seqLen * kvHeads * h.headDim;
    return kvType == 0 ? 2 * values : values + values / 16;
}

// Greedy speculative decoding (--draft-model): why `draftTokens` drafts a round cannot run in this configuration, empty when they
// can (the rules of distributed_llama_b200.api.draft_refusal). target / draft: the model headers once read, the draft's read with
// the target's context length.
inline std::string draftRefusal(uint32_t draftTokens, uint32_t nRanks, uint32_t parallel, const ModelHeader *target = nullptr,
                                const ModelHeader *draft = nullptr) {
    if (draftTokens != 1 && draftTokens != 3 && draftTokens != 7) return "--draft-tokens must be 1, 3 or 7";
    if (nRanks > 1) return "--draft-model runs on one GPU only (no --gpus > 1 or --workers)";
    const char *c = std::getenv("DL_COLLECTIVES");
    if (c && std::string(c) == "nccl") return "--draft-model does not support DL_COLLECTIVES=nccl";
    if (parallel > 1) return "--draft-model does not combine with --parallel > 1";
    if (!target || !draft) return "";
    const std::pair<const char *, const ModelHeader *> models[2] = {{"target model", target}, {"draft model", draft}};
    for (const auto &m : models) {
        if (m.second->nExperts > 0)
            return std::string("--draft-model needs dense models: the ") + m.first + " is mixture-of-experts (no batched verify step)";
        if (m.second->weightType != F_Q40)
            return std::string("--draft-model needs q40 weights: the ") + m.first + " has " + floatTypeName(m.second->weightType) + " weights";
    }
    if (target->vocabSize != draft->vocabSize)
        return "--draft-model needs the target's vocabulary: " + std::to_string(target->vocabSize) + " tokens against " +
               std::to_string(draft->vocabSize);
    if (draft->seqLen < target->seqLen)
        return "--draft-model needs a context of at least " + std::to_string(target->seqLen) + " tokens: the draft model has " +
               std::to_string(draft->seqLen);
    return "";
}

// Counters of speculative rounds and the CLIs' summary line.
struct SpecStats {
    uint64_t rounds = 0, drafted = 0, accepted = 0, emitted = 0;
    std::string line() const {
        char buf[160];
        std::snprintf(buf, sizeof(buf), "Speculative: %llu rounds, %llu drafted, %llu accepted (%.1f %%), %.2f tokens/round",
                      (unsigned long long)rounds, (unsigned long long)drafted, (unsigned long long)accepted,
                      drafted ? 100.0 * (double)accepted / (double)drafted : 0.0, rounds ? (double)emitted / (double)rounds : 0.0);
        return buf;
    }
};

class NativeEngine {
public:
    // maxSeqLen == 0: the model's context length. Throws std::runtime_error on unsupported files / CUDA errors.
    // Tensor parallel (nRanks > 1, one process per GPU of one NVSwitch box): this rank uploads only its slice of every matrix
    // (row slices of q/k/v/w1/w3/logits, column slices of wo/w2 gathered on the host; KV heads are replicated when there are more
    // ranks than KV heads), creates its part of the symmetric peer-memory arena (csrc/cuda/comm_vmm.cu: CUDA VMM + NVSwitch
    // multicast, bootstrapped over unix sockets named after `commTag`) and the kernels do their all-reduces over it. `hostBarrier`
    // must synchronise all ranks of the job (it is called between the two bootstrap steps). Every rank then issues the same
    // sequence of prefill / step calls (reference: root + `dllama worker` processes, src/dllama.cpp:260-285).
    // kvType: KV-cache storage, 0 = bf16, 1 = q80 (EngineConfig::kvType; parseKvCacheFloatType).
    NativeEngine(const std::string &modelPath, uint32_t maxSeqLen, int device, uint32_t rank = 0, uint32_t nRanks = 1,
                 const std::string &commTag = std::string(), std::function<void()> hostBarrier = std::function<void()>(), uint32_t kvType = 0);
    ~NativeEngine();
    NativeEngine(const NativeEngine &) = delete;
    NativeEngine &operator=(const NativeEngine &) = delete;

    const ModelHeader &header() const { return h_; }
    uint32_t seqLen() const { return seqLen_; }
    uint32_t kvType() const { return kvType_; }
    uint64_t bytesUploaded() const { return bytesUploaded_; }
    uint32_t rank() const { return rank_; }
    uint32_t nRanks() const { return nRanks_; }
    bool multicast() const { return multicast_; }
    bool persistentKernel() const { return mega_; }

    // Feeds prompt tokens at positions [pos, pos + n), chunked by the engine (dl_engine_prefill): up to 192 tokens a chunk on
    // the tensor-core path, power-of-two batches of up to 8 on the GEMV path. No logits are produced.
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos);
    // One token; returns the logits row (host memory owned by the engine, valid until the next call). Single GPU only: under tensor
    // parallelism the logits stay sharded on the devices (use stepGreedy / stepSampled).
    const float *step(int32_t token, uint32_t pos);
    // One greedy step entirely on the device (graph replay); returns the next token.
    int32_t stepGreedy(int32_t token, uint32_t pos);
    // One step with temperature / top-p sampling on the device (csrc/cuda/sampler.cu; same xorshift* stream as dl::Sampler). Every
    // rank must have called seedSampler with the same seed; under tensor parallelism every rank draws the same token.
    void seedSampler(uint64_t seed);
    int32_t stepSampled(int32_t token, uint32_t pos, float temperature, float topp);
    uint64_t samplerState();   // single-sequence generator state: seedSampler(samplerState()) continues its stream
    // Presence / frequency penalties and logit bias ((id, value) pairs) of the following device draws; zeroes the count rows in
    // rowMask (bit 0: stepSampled, bit 1 + i: choice i). All zero: off. With controls on, stepSampled and the choices steps accept
    // temperature 0 (arg-max of the controlled logits). Every rank must make the same call.
    void setSamplingControls(float presence, float frequency, const std::vector<std::pair<int32_t, float>> &bias, uint32_t rowMask);
    // top_k / min_p (dl::Sampler::setFilters) of the following sampled device draws of stepSampled and the choices; 0 / 0: off.
    // They persist until changed. Every rank must make the same call.
    void setSamplingFilters(uint32_t topK, float minP);
    // Several completions of one prompt (csrc/cuda/attn_decode.cu), dense models, n <= 8: generators of the batched sampler (separate
    // from the single-sequence one), first draws from the logits of `token` at P, one batched step (see InferenceBackend).
    bool supportsChoices(uint32_t n) const { return n >= 1 && n <= maxBatch_ && h_.nExperts == 0; }
    void seedChoiceSamplers(const std::vector<uint64_t> &seeds);
    std::vector<int32_t> choicesFirst(int32_t token, uint32_t P, uint32_t n, float temperature, float topp);
    std::vector<int32_t> choicesStep(const std::vector<int32_t> &tokens, uint32_t P, uint32_t C, uint32_t j, uint32_t activeMask, float temperature,
                                     float topp);
    // KV-cache slots (csrc/cuda/attn_decode.cu): n <= 8 independent sequences, each in its own floor(seqLen / n) rows of the cache, decoded
    // together by slotsStep. Single GPU, dense q40 models. Row b of a step is slot b (activeMask bit b); inactive rows return -1.
    // paged: the slots share the cache as one pool of 64-row pages instead (engine_api.h: dl_engine_set_slot_cache); slotLen() is
    // then 64 * floor(seqLen / 64) and a slot's rows are reserved before they are written.
    void setSlots(uint32_t n, bool paged = false);
    uint32_t slotLen() const;
    bool slotReserve(uint32_t slot, uint32_t rows);   // false: the pool is short (nothing changed)
    void slotTrim(uint32_t slot, uint32_t rows);
    void slotRelease(uint32_t slot);
    uint32_t freePages() const;
    uint32_t slotPageCount(uint32_t slot) const;
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos);
    void slotCopy(uint32_t src, uint32_t dst, uint32_t P);
    void slotSampling(uint32_t slot, uint64_t seed, float temperature, float topp, float presence, float frequency,
                      const std::vector<std::pair<int32_t, float>> &bias);
    void slotFilters(uint32_t slot, uint32_t topK, float minP);   // off again after every slotSampling
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask);
    // Log-probabilities (csrc/cuda/logprobs.cu, one GPU): setLogprobs(k) makes the following stepGreedy / stepSampled / choicesFirst /
    // choicesStep also compute them for their draws (k top entries, -1: off); logprobsBlocks() holds the result blocks of the last
    // such call, kApiLogprobsWords int32 words per row (engine_api.h). logprobsHostDraw computes them for a token a host Sampler drew
    // from the logits of the last step() (its bias and its counts after the draw are uploaded). slotsStepLogprobs is slotsStep that
    // also fills `blocks` ([slots][kApiLogprobsWords]) for the active slots whose logprobs are on (slotLogprobs).
    void setLogprobs(int k) { lpK_ = k; }
    int logprobs() const { return lpK_; }
    const std::vector<int32_t> &logprobsBlocks() const { return lpHost_; }
    void logprobsHostDraw(int32_t token, uint32_t n, const std::vector<float> &bias, const std::vector<uint32_t> &counts, float presence,
                          float frequency);
    void slotLogprobs(uint32_t slot, int k);
    std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask,
                                           std::vector<int32_t> &blocks);
    // n greedy steps back to back on the device without host round trips; returns the generated tokens.
    std::vector<int32_t> decodeGreedy(int32_t firstToken, uint32_t pos, uint32_t nSteps);
    // One round of greedy speculative decoding with this engine as the target (dl_spec_round): `token` is the last emitted token at
    // `pos`, both engines hold every row before it; the draft proposes k (1, 3, 7; fewer near the end of the context) tokens.
    // Returns the tokens greedy decoding emits next (1 to k + 1) and adds the round to `stats`.
    std::vector<int32_t> specRound(NativeEngine &draft, int32_t token, uint32_t pos, uint32_t k, SpecStats &stats);
    void synchronize();
    // Traffic / synchronisation accounting of the reference's Eval / Pred lines (src/dllama.cpp:59-66): cumulative ns this rank's
    // decode kernel waited for its peers inside the fused all-reduces, and (sent, received) NVLink bytes of a forward over nTokens
    // tokens (2 all-reduces per layer, 8-byte LL words; one multicast store per value when the NVSwitch mapping exists).
    uint64_t syncNs() const;
    void linkBytes(uint32_t nTokens, uint64_t &sent, uint64_t &received) const;
    // Greedy decoding on the device ignores vocabulary rows >= limit (tokenizer vocabulary smaller than the embedding table).
    void setVocabLimit(uint32_t limit);

private:
    struct Impl;
    void *dev(size_t bytes);            // zero-initialised device allocation owned by the engine
    void release();
    void uploadWeights(const uint8_t *file);
    void setInputs(const int32_t *tokens, uint32_t n, uint32_t pos);
    void forward(uint32_t n, int logitsMode, bool greedyAdvance);
    void logprobsAfterDraw(uint32_t rows, uint32_t rowMask, int firstRow, int flags);   // enqueue + copy the blocks, before the sync

    int lpK_ = -1;
    int32_t *lpDev_ = nullptr;
    uint8_t *lpScratch_ = nullptr;
    std::vector<int32_t> lpHost_;

    ModelHeader h_;
    std::vector<TensorEntry> dir_;
    uint32_t slots_ = 1;
    uint32_t seqLen_ = 0, maxBatch_ = 8, nSplits_ = 1, qkvDim_ = 0;
    uint32_t kvType_ = 0;                                                  // KV-cache storage: 0 = bf16, 1 = q80
    uint32_t rank_ = 0, nRanks_ = 1, kvRank_ = 0, kvSlices_ = 1;          // tensor-parallel placement of this process
    uint32_t headsL_ = 0, kvHeadsL_ = 0, ffL_ = 0, vocabL_ = 0;          // per-rank slice sizes
    bool mega_ = false, multicast_ = false;
    uint64_t bytesUploaded_ = 0;
    Impl *impl_ = nullptr;
};

}  // namespace dl
