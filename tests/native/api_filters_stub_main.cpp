// CPU-only harness for the sampling filters (top_k / min_p) of csrc/app/api_server.cpp: the real HTTP / JSON / validation code
// over a fake model whose logits are a fixed function of (token, position, vocabulary id), drawn by the sampler the server hands
// over (single sequence and choices) or by one host Sampler per KV-cache slot built from the slot's settings (--parallel).
// EOS comes `eos-after` positions after the prompt.
// Prints "FLT <top_k> <min_p>" whenever a new completion starts drawing, "SEED <slot> <seed>" for every slotSampling and
// "SLOTFLT <slot> <top_k> <min_p>" for every slotFilters, so the tests can check which filters reached the backend;
// tests/test_sampling_filters.py runs its Python twin through the Python server.
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct FiltersStub : InferenceBackend {
    uint32_t vocab = 0, seq = 4096, eosAfter = 12, prefillEnd = 0, nSlots = 0;
    int32_t eos = 0;
    uint64_t lastCompletion = 0;
    std::vector<float> logits;
    std::vector<std::unique_ptr<Sampler>> slotSampler;
    std::vector<uint32_t> slotStart;
    uint32_t seqLen() const override { return seq; }
    uint32_t vocabSize() const override { return vocab; }
    void fill(int32_t token, uint32_t pos, uint32_t n) {
        logits.resize(n);
        for (uint32_t t = 0; t < n; t++) logits[t] = (float)((t * 2654435761u + (uint32_t)token * 97u + pos * 13u) % 1000u) / 100.0f;
    }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %zu\n", pos, tokens.size());
        prefillEnd = pos + (uint32_t)tokens.size();
    }
    int32_t next(int32_t token, uint32_t pos, Sampler &s) override {
        if (s.completionGeneration() != lastCompletion) {
            lastCompletion = s.completionGeneration();
            std::printf("FLT %u %.9g\n", s.topK(), s.minP());
        }
        if (pos + 1 - prefillEnd > eosAfter) return eos;
        fill(token, pos, s.vocabSize());
        return s.sample(logits.data());
    }
    uint32_t slots() const override { return nSlots; }
    uint32_t slotLen() const override { return nSlots ? seq / nSlots : 0; }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %u %zu\n", slot, pos, tokens.size());
        slotStart[slot] = pos + (uint32_t)tokens.size();
    }
    void slotCopy(uint32_t src, uint32_t dst, uint32_t) override { slotStart[dst] = slotStart[src]; }
    void slotSampling(uint32_t slot, uint64_t seed, float temperature, float topp, float presence, float frequency,
                      const std::vector<std::pair<int32_t, float>> &bias) override {
        std::printf("SEED %u %llu\n", slot, (unsigned long long)seed);
        slotSampler[slot].reset(new Sampler(vocab, temperature, topp, seed));
        slotSampler[slot]->setControls(presence, frequency, bias);
    }
    void slotFilters(uint32_t slot, uint32_t topK, float minP) override {
        std::printf("SLOTFLT %u %u %.9g\n", slot, topK, minP);
        slotSampler[slot]->setFilters(topK, minP);
    }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask) override {
        std::vector<int32_t> out(nSlots, -1);
        for (uint32_t s = 0; s < nSlots; s++) {
            if (!((activeMask >> s) & 1u)) continue;
            if ((uint32_t)pos[s] + 1 - slotStart[s] > eosAfter) { out[s] = eos; continue; }
            fill(tokens[s], (uint32_t)pos[s], vocab);
            out[s] = slotSampler[s]->sample(logits.data());
        }
        return out;
    }
};

int main(int argc, char **argv) {
    if (argc < 4) { std::fprintf(stderr, "usage: api_filters_stub <tokenizer.t> <port> <max-requests> [parallel] [--top-k k] [--min-p p]\n"); return 2; }
    Tokenizer tok(argv[1]);
    FiltersStub b;
    b.vocab = tok.vocabSize();
    b.eos = tok.data().eosIds.at(0);
    ApiConfig cfg;
    cfg.host = "127.0.0.1";
    cfg.port = std::atoi(argv[2]);
    cfg.maxRequests = std::atoi(argv[3]);
    cfg.modelName = "stub.m";
    cfg.temperature = 0.f;
    cfg.parallel = argc > 4 ? (uint32_t)std::atoi(argv[4]) : 1;
    for (int i = 5; i + 1 < argc; i += 2) {
        const std::string name = argv[i];
        if (name == "--top-k") cfg.topK = parseTopK(name, argv[i + 1]);
        else if (name == "--min-p") cfg.minP = parseMinP(name, argv[i + 1]);
    }
    if (cfg.parallel > 1) {
        b.nSlots = cfg.parallel;
        b.slotSampler.resize(b.nSlots);
        b.slotStart.assign(b.nSlots, 0);
    }
    ApiServer server(b, tok, cfg);
    server.serve();
    std::fflush(stdout);
    return 0;
}
