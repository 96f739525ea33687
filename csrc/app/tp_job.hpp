// Process plumbing of a native tensor-parallel job (`dllama-native --gpus N`, `dllama-api-native --gpus N`): one process per GPU
// of one NVSwitch box, forked before CUDA is initialised. Role in the reference: root + `dllama worker` processes and their
// LlmControlPacket stream (src/app.hpp:46-49, src/app.cpp:168-208,306-365) — here the packets travel through a control block in
// an anonymous shared mapping instead of TCP sockets, and a process that dies is noticed by its peers (waitpid / getppid /
// failedRank) instead of hanging them.
#pragma once
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <csignal>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "../host/text.hpp"
#include "native_engine.hpp"

namespace dl {

enum : uint32_t { TP_OP_PREFILL = 1, TP_OP_STEP_GREEDY = 2, TP_OP_STEP_SAMPLED = 3, TP_OP_EXIT = 4, TP_OP_SEED = 5,
                  TP_OP_CHOICES_SEED = 6, TP_OP_CHOICES_FIRST = 7, TP_OP_CHOICES_STEP = 8,
                  TP_OP_CONTROLS = 9,     // penalties in (temperature, topp), count-row mask in pos, tokens = (id, bias bits) pairs
                  TP_OP_FILTERS = 10 };   // sampling filters: top_k in pos, min_p in temperature
constexpr uint32_t kTpMaxRanks = 8, kTpCtrlTokens = 256;

struct TpControl {
    std::atomic<uint32_t> seq;                // bumped by the root for every command
    std::atomic<uint32_t> ack[kTpMaxRanks];   // last command completed by rank r
    std::atomic<uint32_t> arrived;            // bootstrap barrier: monotonic arrival counter
    std::atomic<int32_t> failedRank;          // rank + 1 of the first process that failed, 0 = none
    uint32_t op, n, pos;
    float temperature, topp;
    uint64_t seed;
    int32_t tokens[kTpCtrlTokens];
    char error[240];
};

struct TpJob {   // one process's view of the job
    TpControl *ctl = nullptr;
    uint32_t rank = 0, nRanks = 1, barriers = 0;
    pid_t parentPid = 0;          // the process whose disappearance ends this one (root or supervisor)
    bool reapChildren = false;    // this process forked the other ranks (CLI root): a reaped child = a dead worker
    std::string tag;              // names the bootstrap sockets of the peer-memory arena

    static double nowMs() {
        using namespace std::chrono;
        return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
    }
    // Control block + arena tag; call before forking.
    void create(uint32_t ranks) {
        nRanks = ranks < 1 ? 1 : (ranks > kTpMaxRanks ? kTpMaxRanks : ranks);
        if (nRanks == 1) return;
        void *p = mmap(nullptr, sizeof(TpControl), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
        if (p == MAP_FAILED) throw std::runtime_error("cannot map the control block");
        ctl = new (p) TpControl();
        static int jobs = 0;
        tag = "dllama-" + std::to_string((long)getpid()) + "-" + std::to_string((long long)std::time(nullptr)) + "-" + std::to_string(jobs++);
    }
    void fail(const std::string &what) {
        if (!ctl) return;
        int32_t none = 0;
        if (ctl->failedRank.compare_exchange_strong(none, (int32_t)rank + 1)) std::snprintf(ctl->error, sizeof(ctl->error), "%s", what.c_str());
    }
    void checkPeers() {
        const int32_t f = ctl->failedRank.load();
        if (f != 0 && f != (int32_t)rank + 1) throw std::runtime_error("rank " + std::to_string(f - 1) + " failed: " + std::string(ctl->error));
        if (reapChildren) {
            int st = 0;
            if (waitpid(-1, &st, WNOHANG) > 0) throw std::runtime_error("a worker process exited unexpectedly");
        } else if (parentPid && getppid() != parentPid) {
            throw std::runtime_error("the parent process is gone");
        }
    }
    // spins while the job is active, sleeps between probes after 1 s of waiting (the reference's "turbo off")
    template <typename Pred> void waitFor(Pred done) {
        const double t0 = nowMs();
        for (uint32_t i = 0; !done(); i++) {
            if ((i & 1023u) == 1023u) {
                checkPeers();
                if (nowMs() - t0 > 1000.0) usleep(200);
            }
        }
    }
    void barrier() {   // all ranks, bootstrap only
        barriers++;
        ctl->arrived.fetch_add(1);
        const uint32_t target = barriers * nRanks;
        waitFor([&] { return ctl->arrived.load() >= target; });
    }
    // root: publish a command once every worker has finished the previous one
    void issue(uint32_t op, const int32_t *tokens, uint32_t n, uint32_t pos, float temperature = 0.f, float topp = 0.f, uint64_t seed = 0) {
        if (nRanks == 1) return;
        const uint32_t cur = ctl->seq.load();
        waitFor([&] { for (uint32_t r = 1; r < nRanks; r++) if (ctl->ack[r].load() != cur) return false; return true; });
        ctl->op = op; ctl->n = n; ctl->pos = pos; ctl->temperature = temperature; ctl->topp = topp; ctl->seed = seed;
        for (uint32_t i = 0; i < n && i < kTpCtrlTokens; i++) ctl->tokens[i] = tokens[i];
        ctl->seq.store(cur + 1, std::memory_order_release);
    }
    void sendExit() {
        if (!ctl) return;
        ctl->op = TP_OP_EXIT;
        ctl->seq.store(ctl->seq.load() + 1, std::memory_order_release);
    }
};

// Root-side engine calls of a job: every call is announced to the workers first, then executed locally (the kernels of all ranks
// meet inside their all-reduces).
struct TpEngine {
    NativeEngine &engine;
    TpJob &job;
    uint64_t seedGen = ~0ull, seedOf = 0;   // (generation, seed) of the sampler the device generator was last seeded for
    uint64_t savedGen = ~0ull, savedSeed = 0;
    std::vector<float> hostLogits = {};     // the host sampler's copy of the logits (one GPU)
    uint64_t controlsGen = 0;               // completion generation whose controls the devices hold for stepSampled (0: off)
    uint32_t filtersTopK = 0;               // the sampling filters every rank holds
    float filtersMinP = 0.f;
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) {
        for (size_t i = 0; i < tokens.size(); i += 192) {   // one control packet per tensor-core chunk
            const uint32_t n = (uint32_t)std::min<size_t>(192, tokens.size() - i);
            job.issue(TP_OP_PREFILL, tokens.data() + i, n, pos + (uint32_t)i);
            engine.prefill(std::vector<int32_t>(tokens.begin() + i, tokens.begin() + i + n), pos + (uint32_t)i);
        }
    }
    int32_t stepGreedy(int32_t token, uint32_t pos) {
        job.issue(TP_OP_STEP_GREEDY, &token, 1, pos);
        return engine.stepGreedy(token, pos);
    }
    // One generated token with the sampler's settings: greedy on the device, temperature / top-p on the device under tensor
    // parallelism (the logits stay sharded), or the host sampler on the logits copied back from one GPU.
    // Greedy with sampling controls is the arg-max of the controlled logits (device sampler or host sampler), not the fused arg-max.
    int32_t next(int32_t token, uint32_t pos, Sampler &sampler) {
        if (sampler.temperature() == 0.f && !sampler.controlsActive()) return stepGreedy(token, pos);
        if (engine.nRanks() > 1) return stepSampled(token, pos, sampler);
        const float *logits = engine.step(token, pos);
        hostLogits.assign(logits, logits + sampler.vocabSize());
        const int32_t t = sampler.sample(hostLogits.data());
        if (engine.logprobs() >= 0) {   // the device kernel on the device logits, with this sampler's controls
            std::vector<float> bias;
            if (sampler.controlsActive() && !sampler.logitBias().empty()) {
                bias.assign(sampler.vocabSize(), 0.f);
                for (const auto &b : sampler.logitBias()) bias[(size_t)b.first] = b.second;
            }
            engine.logprobsHostDraw(t, sampler.vocabSize(), bias, sampler.controlsActive() ? sampler.counts() : std::vector<uint32_t>(),
                                    sampler.presencePenalty(), sampler.frequencyPenalty());
        }
        return t;
    }
    // temperature / top-p on the device (the logits stay sharded); `sampler` only supplies the parameters and the seed
    int32_t stepSampled(int32_t token, uint32_t pos, Sampler &sampler) {
        const uint64_t gen = sampler.controlsActive() ? sampler.completionGeneration() : 0;
        if (gen != controlsGen) {   // a new completion: count row 0 starts from zero
            setControls(sampler, 1u);
            controlsGen = gen;
        }
        setFilters(sampler);
        if (sampler.temperature() != 0.f && (sampler.seedGeneration() != seedGen || sampler.seed() != seedOf)) {
            seedGen = sampler.seedGeneration();
            seedOf = sampler.seed();
            job.issue(TP_OP_SEED, nullptr, 0, 0, 0.f, 0.f, sampler.seed());
            engine.seedSampler(sampler.seed());
        }
        job.issue(TP_OP_STEP_SAMPLED, &token, 1, pos, sampler.temperature(), sampler.topp());
        return engine.stepSampled(token, pos, sampler.temperature(), sampler.topp());
    }
    void setControls(const Sampler &sampler, uint32_t rowMask) {
        std::vector<int32_t> w;
        for (const auto &b : sampler.logitBias()) {
            uint32_t bits;
            std::memcpy(&bits, &b.second, 4);
            w.push_back(b.first);
            w.push_back((int32_t)bits);
        }
        job.issue(TP_OP_CONTROLS, w.data(), (uint32_t)w.size(), rowMask, sampler.presencePenalty(), sampler.frequencyPenalty());
        engine.setSamplingControls(sampler.presencePenalty(), sampler.frequencyPenalty(), sampler.logitBias(), rowMask);
    }
    // The sampler's top_k / min_p on every rank before the first draw that uses them: each rank draws from the gathered logits
    // with its own generator, so all ranks must hold the same filters.
    void setFilters(const Sampler &sampler) {
        if (sampler.topK() == filtersTopK && sampler.minP() == filtersMinP) return;
        job.issue(TP_OP_FILTERS, nullptr, 0, sampler.topK(), sampler.minP());
        engine.setSamplingFilters(sampler.topK(), sampler.minP());
        filtersTopK = sampler.topK();
        filtersMinP = sampler.minP();
    }
    // the batched choices' controls (count rows 1..n zeroed) and filters
    void choiceControls(const Sampler &sampler, uint32_t n) {
        setFilters(sampler);
        if (!sampler.controlsActive() && controlsGen == 0) return;
        setControls(sampler, ((1u << n) - 1u) << 1);
        controlsGen = sampler.controlsActive() ? ~0ull : 0;   // row 0's counts are not this sampler's
    }
    // the single-sequence generator's state, and re-seeding every rank with it (sequential choices re-seed it per choice)
    uint64_t samplerState() {
        savedGen = seedGen; savedSeed = seedOf;
        return seedGen == ~0ull ? 0 : engine.samplerState();
    }
    void restoreSampler(uint64_t state) {
        seedGen = savedGen; seedOf = savedSeed;
        if (seedGen == ~0ull) return;   // never seeded before the request: the next sampled step seeds afresh
        job.issue(TP_OP_SEED, nullptr, 0, 0, 0.f, 0.f, state);
        engine.seedSampler(state);
    }
    // choices: seeds travel as (lo, hi) token pairs; step packets carry [C, j, activeMask, tokens...]
    void seedChoices(const std::vector<uint64_t> &seeds) {
        std::vector<int32_t> w;
        for (uint64_t s : seeds) { w.push_back((int32_t)(uint32_t)s); w.push_back((int32_t)(uint32_t)(s >> 32)); }
        job.issue(TP_OP_CHOICES_SEED, w.data(), (uint32_t)w.size(), 0);
        engine.seedChoiceSamplers(seeds);
    }
    std::vector<int32_t> choicesFirst(int32_t token, uint32_t P, uint32_t n, float temperature, float topp) {
        const int32_t w[2] = {token, (int32_t)n};
        job.issue(TP_OP_CHOICES_FIRST, w, 2, P, temperature, topp);
        return engine.choicesFirst(token, P, n, temperature, topp);
    }
    std::vector<int32_t> choicesStep(const std::vector<int32_t> &tokens, uint32_t P, uint32_t C, uint32_t j, uint32_t activeMask, float temperature,
                                     float topp) {
        std::vector<int32_t> w = {(int32_t)C, (int32_t)j, (int32_t)activeMask};
        w.insert(w.end(), tokens.begin(), tokens.end());
        job.issue(TP_OP_CHOICES_STEP, w.data(), (uint32_t)w.size(), P, temperature, topp);
        return engine.choicesStep(tokens, P, C, j, activeMask, temperature, topp);
    }
};

// Bias pairs of a TP_OP_CONTROLS packet.
inline std::vector<std::pair<int32_t, float>> tpControlBias(const int32_t *w, uint32_t n) {
    std::vector<std::pair<int32_t, float>> bias;
    for (uint32_t i = 0; i + 1 < n; i += 2) {
        float v;
        std::memcpy(&v, &w[i + 1], 4);
        bias.push_back({w[i], v});
    }
    return bias;
}

// Seeds of a TP_OP_CHOICES_SEED packet.
inline std::vector<uint64_t> tpChoiceSeeds(const int32_t *w, uint32_t n) {
    std::vector<uint64_t> seeds;
    for (uint32_t i = 0; i + 1 < n; i += 2) seeds.push_back((uint64_t)(uint32_t)w[i] | ((uint64_t)(uint32_t)w[i + 1] << 32));
    return seeds;
}

// ranks >= 1: mirror the root's engine calls until TP_OP_EXIT (reference: runWorkerApp, src/app.cpp:306-365). Returns the exit code.
inline int tpWorkerMain(const std::string &model, const std::string &tokenizer, uint32_t maxSeqLen, int gpuIndex, TpJob &job,
                        uint32_t kvType = 0) {
    try {
        NativeEngine engine(model, maxSeqLen, gpuIndex + (int)job.rank, job.rank, job.nRanks, job.tag, [&job] { job.barrier(); }, kvType);
        {
            Tokenizer tok(tokenizer);      // only for the vocabulary limit of the greedy arg-max (must match the root)
            engine.setVocabLimit(tok.vocabSize());
        }
        job.barrier();                     // "weights loaded" on every rank
        uint32_t mine = 0;
        while (true) {
            job.waitFor([&] { return job.ctl->seq.load(std::memory_order_acquire) != mine; });
            mine++;
            const TpControl &c = *job.ctl;
            if (c.op == TP_OP_EXIT) break;
            if (c.op == TP_OP_PREFILL) { engine.prefill(std::vector<int32_t>(c.tokens, c.tokens + c.n), c.pos); engine.synchronize(); }
            else if (c.op == TP_OP_STEP_GREEDY) engine.stepGreedy(c.tokens[0], c.pos);
            else if (c.op == TP_OP_STEP_SAMPLED) engine.stepSampled(c.tokens[0], c.pos, c.temperature, c.topp);
            else if (c.op == TP_OP_SEED) engine.seedSampler(c.seed);
            else if (c.op == TP_OP_CONTROLS) engine.setSamplingControls(c.temperature, c.topp, tpControlBias(c.tokens, c.n), c.pos);
            else if (c.op == TP_OP_FILTERS) engine.setSamplingFilters(c.pos, c.temperature);
            else if (c.op == TP_OP_CHOICES_SEED) engine.seedChoiceSamplers(tpChoiceSeeds(c.tokens, c.n));
            else if (c.op == TP_OP_CHOICES_FIRST) engine.choicesFirst(c.tokens[0], c.pos, (uint32_t)c.tokens[1], c.temperature, c.topp);
            else if (c.op == TP_OP_CHOICES_STEP)
                engine.choicesStep(std::vector<int32_t>(c.tokens + 3, c.tokens + c.n), c.pos, (uint32_t)c.tokens[0], (uint32_t)c.tokens[1],
                                   (uint32_t)c.tokens[2], c.temperature, c.topp);
            job.ctl->ack[job.rank].store(mine, std::memory_order_release);
        }
        job.ctl->ack[job.rank].store(mine, std::memory_order_release);
        return 0;
    } catch (const std::exception &e) {
        job.fail(e.what());
        return 1;
    }
}

// Ends a set of child processes: 3 s of grace after the exit command, then SIGKILL.
inline void tpReap(std::vector<pid_t> &children) {
    for (pid_t c : children) {
        if (c <= 0) continue;
        bool gone = false;
        for (int i = 0; i < 3000 && !gone; i++) {
            int st = 0;
            if (waitpid(c, &st, WNOHANG) != 0) gone = true; else usleep(1000);
        }
        if (!gone) { kill(c, SIGKILL); waitpid(c, nullptr, 0); }
    }
    children.clear();
}

}  // namespace dl
