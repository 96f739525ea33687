// CPU-only harness for the --parallel server of csrc/app/api_server.cpp: the real HTTP / JSON / template / stop-detector / per-slot
// NaiveCache / scheduling code over a fake slot backend. A row's next token is a fixed function of (token, position, and its
// slot's seed when sampling), never of the slot index or the other rows; EOS comes after `eos-after` tokens of a completion. Every
// step sleeps `delay-ms`, so that requests overlap in time. A row's log-probability entry is a fixed float32 function of (drawn
// token, position, k). The Python twin is SlotStub in tests/test_api_parallel.py.
// Prints "POS <slot> <start> <n>" for every prefill, "COPY <src> <dst> <P>" for every prompt copy and "SEED <slot> <seed>" for
// every slotSampling.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct SlotStub : InferenceBackend {
    uint32_t vocab = 0, regular = 0, n = 4, len = 256, eosAfter = 10, delayMs = 20;
    int32_t eos = 0;
    std::vector<uint64_t> seed;
    std::vector<float> temp;
    std::vector<uint32_t> produced;
    std::vector<int> k;   // top_logprobs of each slot's draws, -1: none
    uint32_t seqLen() const override { return n * len; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &, uint32_t) override { throw std::runtime_error("single-sequence call in --parallel mode"); }
    int32_t next(int32_t, uint32_t, Sampler &) override { throw std::runtime_error("single-sequence call in --parallel mode"); }
    uint32_t slots() const override { return n; }
    uint32_t slotLen() const override { return len; }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %u %zu\n", slot, pos, tokens.size());
    }
    void slotCopy(uint32_t src, uint32_t dst, uint32_t P) override { std::printf("COPY %u %u %u\n", src, dst, P); }
    void slotSampling(uint32_t slot, uint64_t s, float temperature, float, float, float, const std::vector<std::pair<int32_t, float>> &) override {
        std::printf("SEED %u %llu\n", slot, (unsigned long long)s);
        seed[slot] = s;
        temp[slot] = temperature;
        produced[slot] = 0;
        k[slot] = -1;
    }
    void slotLogprobs(uint32_t slot, int kk) override { k[slot] = kk; }
    std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask,
                                           std::vector<TokenLogprobs> &rows) override {
        const std::vector<int32_t> out = slotsStep(tokens, pos, activeMask);
        rows.assign(n, TokenLogprobs());
        for (uint32_t b = 0; b < n; b++) {
            if (!((activeMask >> b) & 1u) || k[b] < 0) continue;
            TokenLogprobs &e = rows[b];
            e.token = out[b];
            e.logprob = -(float)(pos[b] % 7) * 0.37f;
            for (int j = 0; j < k[b]; j++) e.top.push_back({(int32_t)((out[b] + 31 * j) % regular), -(float)j * 0.2517f - 0.001f});
        }
        return out;
    }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask) override {
        std::this_thread::sleep_for(std::chrono::milliseconds(delayMs));
        std::vector<int32_t> out(n, -1);
        for (uint32_t b = 0; b < n; b++) {
            if (!((activeMask >> b) & 1u)) continue;
            const uint64_t salt = temp[b] > 0.f ? (seed[b] % 997u) * 31u : 0u;
            out[b] = ++produced[b] > eosAfter ? eos : (int32_t)(((uint64_t)tokens[b] * 7u + (uint64_t)pos[b] * 13u + 5u + salt) % regular);
        }
        return out;
    }
};

int main(int argc, char **argv) {
    if (argc < 5) {
        std::fprintf(stderr, "usage: api_parallel_stub <tokenizer.t> <port> <max-requests> <parallel> [eos-after] [delay-ms] [seed]\n");
        return 2;
    }
    Tokenizer tok(argv[1]);
    SlotStub b;
    b.vocab = tok.vocabSize();
    b.regular = tok.regularVocabSize();
    b.eos = tok.data().eosIds.at(0);
    b.n = (uint32_t)std::atoi(argv[4]);
    b.len = 1024 / b.n;
    b.eosAfter = argc > 5 ? (uint32_t)std::atoi(argv[5]) : 10;
    b.delayMs = argc > 6 ? (uint32_t)std::atoi(argv[6]) : 20;
    b.seed.assign(b.n, 0);
    b.temp.assign(b.n, 0.f);
    b.produced.assign(b.n, 0);
    b.k.assign(b.n, -1);
    ApiConfig cfg;
    cfg.host = "127.0.0.1";
    cfg.port = std::atoi(argv[2]);
    cfg.maxRequests = std::atoi(argv[3]);
    cfg.modelName = "stub.m";
    cfg.temperature = 0.f;
    cfg.seed = argc > 7 ? std::strtoull(argv[7], nullptr, 10) : 77;
    cfg.parallel = b.n;
    ApiServer server(b, tok, cfg);
    server.serve();
    return 0;
}
