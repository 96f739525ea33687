// CPU-only harness for the sampling controls of csrc/app/api_server.cpp: the real HTTP / JSON / validation code over a fake model
// whose logits are a fixed function of (token, position, vocabulary id), drawn by the sampler the server hands over (the host
// Sampler with the request's controls). EOS comes `eos-after` positions after the prefilled prompt.
// Prints "CTL <presence> <frequency> <id>:<bias> ..." whenever a new completion starts drawing, so the tests can check which controls
// reached the backend; tests/test_sampling_controls.py runs its Python twin through the Python server.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct ControlsStub : InferenceBackend {
    uint32_t vocab, seq, eosAfter, prefillEnd = 0;
    int32_t eos;
    uint64_t lastCompletion = 0;
    std::vector<float> logits;
    uint32_t seqLen() const override { return seq; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %zu\n", pos, tokens.size());
        prefillEnd = pos + (uint32_t)tokens.size();
    }
    int32_t next(int32_t token, uint32_t pos, Sampler &s) override {
        if (s.completionGeneration() != lastCompletion) {
            lastCompletion = s.completionGeneration();
            std::printf("CTL %.9g %.9g", s.presencePenalty(), s.frequencyPenalty());
            for (const auto &b : s.logitBias()) std::printf(" %d:%.9g", b.first, b.second);
            std::printf("\n");
        }
        if (pos + 1 - prefillEnd > eosAfter) return eos;
        logits.resize(s.vocabSize());
        for (uint32_t t = 0; t < s.vocabSize(); t++)
            logits[t] = (float)((t * 2654435761u + (uint32_t)token * 97u + pos * 13u) % 1000u) / 100.0f;
        return s.sample(logits.data());
    }
};

int main(int argc, char **argv) {
    if (argc < 4) { std::fprintf(stderr, "usage: api_controls_stub <tokenizer.t> <port> <max-requests> [eos-after]\n"); return 2; }
    Tokenizer tok(argv[1]);
    ControlsStub b;
    b.vocab = tok.vocabSize();
    b.seq = 4096;
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
    std::fflush(stdout);
    return 0;
}
