// `dllama-api-native`: the OpenAI-style HTTP server of the reference (src/dllama-api.cpp:602-632) as a native binary on one
// GPU — api_server.cpp (HTTP, JSON, NaiveCache, templates, stop detection) over NativeEngine. Multi-GPU serving: ./dllama-api --gpus N.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <ctime>
#include <stdexcept>
#include <string>
#include <thread>

#include "api_server.hpp"
#include <sys/prctl.h>

#include "../cuda/engine_api.h"
#include "native_engine.hpp"
#include "tp_job.hpp"

using namespace dl;

namespace {

struct EngineBackend : InferenceBackend {
    NativeEngine &e;
    TpEngine tp;              // announces every engine call to the worker ranks of a --gpus N job (no-op on one GPU)
    EngineBackend(NativeEngine &engine, TpJob &job) : e(engine), tp{engine, job} {}
    uint32_t seqLen() const override { return e.seqLen(); }
    uint32_t vocabSize() const override { return e.header().vocabSize; }
    void setVocabLimit(uint32_t limit) override {
        e.setVocabLimit(limit);
        if (draft) draft->setVocabLimit(limit);
    }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override {
        if (tokens.empty()) return;
        tp.prefill(tokens, pos);
        if (draft) draft->prefill(tokens, pos);   // the draft follows every prefill, prompt-cache continuations included
    }
    int32_t next(int32_t token, uint32_t pos, Sampler &sampler) override { return tp.next(token, pos, sampler); }
    // --draft-model (one GPU): greedy single completions decode in speculative rounds
    NativeEngine *draft = nullptr;
    uint32_t draftTokens = 3;
    SpecStats specStats;
    bool speculates(const Sampler &sampler) const override { return draft && sampler.temperature() == 0.f && !sampler.controlsActive(); }
    std::vector<int32_t> specRound(int32_t token, uint32_t pos) override { return e.specRound(*draft, token, pos, draftTokens, specStats); }
    // choices: one batched step per token on dense models; the sequential fallback (MoE) keeps the device generator's stream
    bool batchedChoices(uint32_t n) const override { return e.supportsChoices(n); }
    void seedChoices(const std::vector<uint64_t> &seeds) override { tp.seedChoices(seeds); }
    void choiceControls(const Sampler &sampler, uint32_t n) override { tp.choiceControls(sampler, n); }
    std::vector<int32_t> choicesFirst(int32_t token, uint32_t P, uint32_t n, float temperature, float topp) override {
        return tp.choicesFirst(token, P, n, temperature, topp);
    }
    std::vector<int32_t> choicesStep(const std::vector<int32_t> &tokens, uint32_t P, uint32_t C, uint32_t j, uint32_t activeMask, float temperature,
                                     float topp) override {
        return tp.choicesStep(tokens, P, C, j, activeMask, temperature, topp);
    }
    uint64_t saveSampler() override { return e.nRanks() > 1 ? tp.samplerState() : 0; }
    void restoreSampler(uint64_t saved) override { if (e.nRanks() > 1) tp.restoreSampler(saved); }
    // KV-cache slots (--parallel > 1): one GPU only, so the calls go straight to the engine
    uint32_t slotCount = 0;
    uint32_t slots() const override { return slotCount; }
    uint32_t slotLen() const override { return e.slotLen(); }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) override { e.slotPrefill(slot, tokens, pos); }
    void slotCopy(uint32_t src, uint32_t dst, uint32_t P) override { e.slotCopy(src, dst, P); }
    bool pagedSlots = false;
    bool paged() const override { return pagedSlots; }
    bool slotReserve(uint32_t slot, uint32_t rows) override { return e.slotReserve(slot, rows); }
    void slotTrim(uint32_t slot, uint32_t rows) override { e.slotTrim(slot, rows); }
    void slotRelease(uint32_t slot) override { e.slotRelease(slot); }
    uint32_t freePages() const override { return e.freePages(); }
    uint32_t slotPageCount(uint32_t slot) const override { return e.slotPageCount(slot); }
    void slotSampling(uint32_t slot, uint64_t seed, float temperature, float topp, float presence, float frequency,
                      const std::vector<std::pair<int32_t, float>> &bias) override {
        e.slotSampling(slot, seed, temperature, topp, presence, frequency, bias);
    }
    void slotFilters(uint32_t slot, uint32_t topK, float minP) override { e.slotFilters(slot, topK, minP); }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask) override {
        return e.slotsStep(tokens, pos, activeMask);
    }
    // log-probabilities: one GPU only (the vocabulary is sliced over the ranks of a --gpus N job)
    void setLogprobs(int k) override {
        if (k >= 0 && e.nRanks() > 1) throw std::runtime_error("logprobs are not supported under tensor parallelism yet");
        e.setLogprobs(k);
    }
    std::vector<TokenLogprobs> lastLogprobs() override {
        const std::vector<int32_t> &w = e.logprobsBlocks();
        std::vector<TokenLogprobs> out;
        for (size_t r = 0; r + kApiLogprobsWords <= w.size(); r += kApiLogprobsWords) out.push_back(decodeLogprobs(w.data() + r));
        return out;
    }
    void slotLogprobs(uint32_t slot, int k) override { e.slotLogprobs(slot, k); }
    std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask,
                                           std::vector<TokenLogprobs> &rows) override {
        std::vector<int32_t> blocks;
        std::vector<int32_t> out = e.slotsStepLogprobs(tokens, pos, activeMask, blocks);
        rows.assign(out.size(), TokenLogprobs());
        for (size_t s = 0; s < out.size(); s++)
            if (blocks[s * kApiLogprobsWords + 2] >= 0) rows[s] = decodeLogprobs(blocks.data() + s * kApiLogprobsWords);
        return out;
    }
};

// A --parallel value this configuration cannot serve: reported in one line, not retried.
struct ParallelRefused : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// Why --parallel `parallel` with slot layout `cache` cannot run here (empty: it can); the rules of distributed_llama_b200.api.parallel_refusal.
std::string parallelRefusal(uint32_t parallel, uint32_t nRanks, uint32_t nExperts, const std::string &cache) {
    if (cache != "split" && cache != "paged") return "--parallel-cache must be split or paged, not '" + cache + "'";
    if (parallel < 1 || parallel > kMaxChoices) return "--parallel must be from 1 to 8";
    if (parallel == 1) return "";
    if (nRanks > 1) return "--parallel > 1 runs on one GPU only (workers cannot mirror slot steps yet)";
    if (nExperts > 0) return "--parallel > 1 does not support mixture-of-experts models (the batched step has no MoE path)";
    const char *c = std::getenv("DL_COLLECTIVES");
    if (c && std::string(c) == "nccl") return "--parallel > 1 does not support DL_COLLECTIVES=nccl";
    if (std::getenv("DL_HOST_SAMPLER")) return "--parallel > 1 samples on the device: unset DL_HOST_SAMPLER";
    return "";
}

const char *kUsage =
    "Usage: dllama-api-native --model <path> --tokenizer <path> [--host <addr>] [--port <p>] [--max-seq-len <n>]\n"
    "        [--temperature <t>] [--topp <p>] [--presence-penalty <p>] [--frequency-penalty <f>] [--seed <s>]\n"
    "        [--top-k <k>] [--min-p <p>]  sampling filters of sampled draws (default 0 = off; requests may override them)\n"
    "        [--chat-template {llama2|llama3|deepSeek3|chatml}] [--gpu-index <i>]\n"
    "        [--kv-cache-float-type {bf16|q80}]  KV-cache storage (default bf16; q80 = int8 blocks of 32 + f16 scale)\n"
    "        [--parallel <n>]  decode up to n (1..8) chat requests together, each in its own KV-cache slot of floor(context / n)\n"
    "                       tokens; one GPU and dense models only\n"
    "        [--parallel-cache {split|paged}]  paged: the slots share the KV cache as one pool of 64-token pages (default split)\n"
    "        [--draft-model <path>] [--draft-tokens {1|3|7}]  greedy single completions decode in speculative rounds: the draft\n"
    "                       (same tokenizer, dense q40) proposes k tokens (default 3), the model checks them in one forward\n"
    "        [--gpus <n>]   tensor parallel over n GPUs: a supervisor forks one process per GPU (rank 0 serves HTTP) and restarts\n"
    "                       the whole job 3 s after any rank fails\n";

// One attempt of rank 0 of a job (or the only process on one GPU): engine + tokenizer + HTTP server until --max-requests is reached.
int serveOnce(const std::string &model, const std::string &tokenizer, uint32_t maxSeqLen, int gpu, const ApiConfig &cfg, TpJob &job,
              uint32_t kvType, const std::string &parallelCache, const std::string &draftModel, uint32_t draftTokens) {
    NativeEngine engine(model, maxSeqLen, gpu, 0, job.nRanks, job.tag, [&job] { job.barrier(); }, kvType);
    Tokenizer tok(tokenizer);
    if (job.nRanks > 1) job.barrier();   // every rank has its weights
    std::printf("%s%s", tok.describe().c_str(), describeModelHeader(engine.header()).c_str());
    if (job.nRanks > 1)
        std::printf("🔗 %u GPUs (one process each), all-reduce inside the kernels over %s\n", job.nRanks,
                    engine.multicast() ? "the NVSwitch multicast mapping (multimem.st)" : "NVLink peer memory");
    std::printf("💿 Weights loaded\n");
    EngineBackend backend(engine, job);
    const std::string why = parallelRefusal(cfg.parallel, job.nRanks, engine.header().nExperts, parallelCache);
    if (!why.empty()) throw ParallelRefused(why);
    std::unique_ptr<NativeEngine> draft;
    if (!draftModel.empty()) {
        // the draft gets the target's context length and KV-cache storage; refused in one line before its weights load
        const ModelHeader dh = loadModelHeader(draftModel, engine.seqLen());
        const std::string whyDraft = draftRefusal(draftTokens, job.nRanks, cfg.parallel, &engine.header(), &dh);
        if (!whyDraft.empty()) throw ParallelRefused(whyDraft);
        draft.reset(new NativeEngine(draftModel, engine.seqLen(), gpu, 0, 1, std::string(), std::function<void()>(), kvType));
        backend.draft = draft.get();
        backend.draftTokens = draftTokens;
    }
    if (cfg.parallel > 1) {
        engine.setSlots(cfg.parallel, parallelCache == "paged");
        backend.slotCount = cfg.parallel;
        backend.pagedSlots = parallelCache == "paged";
    }
    ApiServer server(backend, tok, cfg);
    server.serve();
    return 0;
}

}  // namespace

int main(int argc, char **argv) {
    std::string model, tokenizer;
    ApiConfig cfg;
    cfg.seed = (uint64_t)std::time(nullptr);
    uint32_t maxSeqLen = 0, kvType = 0;
    int gpu = 0;
    uint32_t gpus = 1, workers = 0;
    std::string parallelCache = "split", draftModel;
    uint32_t draftTokens = 3;
    try {
        for (int i = 1; i < argc;) {
            const std::string name = argv[i];
            if (name == "--help" || name == "-h" || name == "--usage") { std::fprintf(stderr, "%s", kUsage); return 0; }
            if (name == "--workers") { i++; while (i < argc && argv[i][0] != '-') { i++; workers++; } continue; }
            if (i + 1 >= argc) throw std::runtime_error("Missing value for " + name);
            const std::string v = argv[i + 1];
            if (name == "--model") model = v;
            else if (name == "--tokenizer") tokenizer = v;
            else if (name == "--host") cfg.host = v;
            else if (name == "--port") cfg.port = std::stoi(v);
            else if (name == "--max-seq-len") maxSeqLen = (uint32_t)std::stoul(v);
            else if (name == "--kv-cache-float-type") kvType = parseKvCacheFloatType(v);
            else if (name == "--temperature") cfg.temperature = std::stof(v);
            else if (name == "--topp") cfg.topp = std::stof(v);
            else if (name == "--presence-penalty") cfg.presencePenalty = parsePenalty(name, v);
            else if (name == "--frequency-penalty") cfg.frequencyPenalty = parsePenalty(name, v);
            else if (name == "--top-k") cfg.topK = parseTopK(name, v);
            else if (name == "--min-p") cfg.minP = parseMinP(name, v);
            else if (name == "--seed") cfg.seed = std::stoull(v);
            else if (name == "--chat-template") cfg.chatTemplate = v;
            else if (name == "--gpu-index") gpu = std::max(0, std::stoi(v));
            else if (name == "--gpus") gpus = (uint32_t)std::max(1, std::stoi(v));
            else if (name == "--max-requests") cfg.maxRequests = std::stoi(v);
            else if (name == "--parallel") cfg.parallel = (uint32_t)std::max(0, std::stoi(v));
            else if (name == "--parallel-cache") parallelCache = v;
            else if (name == "--draft-model") draftModel = v;
            else if (name == "--draft-tokens") draftTokens = (uint32_t)std::max(0, std::stoi(v));
            else if (name == "--buffer-float-type" || name == "--nthreads" || name == "--net-turbo" || name == "--gpu-segments") {}
            else throw std::runtime_error("Unknown option: " + name);
            i += 2;
        }
        if (model.empty()) throw std::runtime_error("Model is required");
        if (tokenizer.empty()) throw std::runtime_error("Tokenizer is required");
    } catch (const std::exception &e) {
        std::printf("🚨 Critical error: %s\n", e.what());
        return 1;
    }
    {
        std::string why = parallelRefusal(cfg.parallel, gpus + workers, 0, parallelCache);
        if (why.empty() && !draftModel.empty()) why = draftRefusal(draftTokens, gpus + workers, cfg.parallel);
        if (!why.empty()) { std::fprintf(stderr, "%s\n", why.c_str()); return 1; }
    }
    const size_t slash = model.find_last_of("/\\");
    cfg.modelName = slash == std::string::npos ? model : model.substr(slash + 1);
    // the reference retries its whole inference app every 3 s on errors (dllama-api.cpp:616-628)
    if (gpus <= 1) {
        while (true) {
            try {
                TpJob job;
                return serveOnce(model, tokenizer, maxSeqLen, gpu, cfg, job, kvType, parallelCache, draftModel, draftTokens);
            } catch (const ParallelRefused &e) {
                std::fprintf(stderr, "%s\n", e.what());
                return 1;
            } catch (const std::exception &e) {
                std::printf("🚨 Inference error: %s\n🔄 Retrying in 3 seconds...\n", e.what());
                std::fflush(stdout);
                std::this_thread::sleep_for(std::chrono::seconds(3));
            }
        }
    }
    // Tensor parallel: this process is a supervisor without a CUDA context, so it can fork a fresh set of ranks for every attempt.
    // Rank 0 serves HTTP, ranks >= 1 mirror its engine calls (tp_job.hpp). The first process that exits ends the attempt: rank 0
    // returning 0 = --max-requests reached; anything else (a rank crashed, a device-side wait timed out, a peer disappeared) tears
    // the job down and a new one is started after 3 s — the reference's root retry loop plus its worker re-listen loop
    // (src/dllama-api.cpp:616-628, src/app.cpp:306-365).
    while (true) {
        TpJob job;
        job.create(gpus);
        const pid_t supervisor = getpid();
        std::vector<pid_t> kids;
        std::fflush(stdout);
        for (uint32_t r = 0; r < job.nRanks; r++) {
            const pid_t pid = fork();
            if (pid < 0) { std::printf("🚨 Critical error: fork failed\n"); return 1; }
            if (pid == 0) {
                prctl(PR_SET_PDEATHSIG, SIGKILL);
                job.rank = r; job.parentPid = supervisor;
                int rc = 1;
                if (r == 0) {
                    try {
                        rc = serveOnce(model, tokenizer, maxSeqLen, gpu, cfg, job, kvType, parallelCache, draftModel, draftTokens);
                        job.sendExit();
                    } catch (const std::exception &e) {
                        job.fail(e.what());
                        std::printf("🚨 Inference error: %s\n", e.what());
                    }
                } else {
                    std::fclose(stdin);
                    rc = tpWorkerMain(model, tokenizer, maxSeqLen, gpu, job, kvType);
                }
                std::fflush(stdout);
                _exit(rc);
            }
            kids.push_back(pid);
        }
        int st = 0;
        const pid_t first = waitpid(-1, &st, 0);
        const bool served = first == kids[0] && WIFEXITED(st) && WEXITSTATUS(st) == 0;
        uint32_t who = 0;
        for (uint32_t r = 0; r < kids.size(); r++) if (kids[r] == first) { who = r; kids[r] = 0; }
        job.sendExit();
        if (!served && kids[0] > 0) kill(kids[0], SIGTERM);   // rank 0 may be blocked in accept()
        tpReap(kids);
        const std::string why = job.ctl && job.ctl->failedRank.load() ? std::string(": ") + job.ctl->error : std::string();
        if (job.ctl) munmap(job.ctl, sizeof(TpControl));
        if (served) return 0;
        std::printf("🚨 Inference error: rank %u ended the job%s\n🔄 Retrying in 3 seconds...\n", who, why.c_str());
        std::fflush(stdout);
        std::this_thread::sleep_for(std::chrono::seconds(3));
    }
}
