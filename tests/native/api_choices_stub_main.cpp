// CPU-only harness for csrc/app/api_server.cpp: the real HTTP / JSON / chat-template / stop-detector / NaiveCache code over a
// deterministic fake model (next token = a fixed function of (token, position); emits EOS after `eos-after` tokens). With a
// temperature above 0 the token also depends on the sampler's seed, so the choices of an `n` request differ, and EOS comes
// `eos-after` positions after the prefilled prompt, so every choice of the sequential path gets the same length.
// Prints "POS <start> <n>" for every prefill so the tests can check the prefix re-use of NaiveCache.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct StubBackend : InferenceBackend {
    uint32_t vocab, regular, seq;
    int32_t eos;
    uint32_t eosAfter, produced = 0, prefillEnd = 0;
    uint32_t seqLen() const override { return seq; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %zu\n", pos, tokens.size());
        produced = 0;
        prefillEnd = pos + (uint32_t)tokens.size();
    }
    int32_t next(int32_t token, uint32_t pos, Sampler &s) override {
        if (s.temperature() > 0.f) {
            if (pos + 1 - prefillEnd > eosAfter) return eos;
            return (int32_t)(((uint64_t)(uint32_t)token * 7u + pos * 13u + 5u + (s.seed() % 997u) * 31u) % regular);
        }
        if (++produced > eosAfter) return eos;
        return (int32_t)(((uint32_t)token * 7u + pos * 13u + 5u) % regular);
    }
};

int main(int argc, char **argv) {
    if (argc < 4) { std::fprintf(stderr, "usage: api_stub <tokenizer.t> <port> <max-requests> [eos-after] [seq-len]\n"); return 2; }
    Tokenizer tok(argv[1]);
    StubBackend b;
    b.vocab = tok.vocabSize();
    b.regular = tok.regularVocabSize();
    b.seq = argc > 5 ? (uint32_t)std::atoi(argv[5]) : 4096;
    b.eos = tok.data().eosIds.at(0);
    b.eosAfter = argc > 4 ? (uint32_t)std::atoi(argv[4]) : 12;
    ApiConfig cfg;
    cfg.host = "127.0.0.1";
    cfg.port = std::atoi(argv[2]);
    cfg.maxRequests = std::atoi(argv[3]);
    cfg.modelName = "stub.m";
    cfg.temperature = 0.f;
    ApiServer server(b, tok, cfg);
    server.serve();
    return 0;
}
