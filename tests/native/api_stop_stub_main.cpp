// CPU-only harness for `stop` strings in csrc/app/api_server.cpp: the model of api_logprobs_stub_main.cpp (logits a fixed function
// of (token, position, vocabulary id) drawn by the host Sampler, end of sequence `eos-after` tokens after the prefilled prompt,
// log-probability entries a fixed float32 function of (drawn token, position, k)) that also prints "POS <start> <n>" for every
// prefill, so that tests/test_stop_sequences.py can check where the prompt cache lets a follow-up start. Its Python twin is
// StopStub there.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct StopStub : InferenceBackend {
    uint32_t vocab = 0, seq = 4096, eosAfter = 12, prefillEnd = 0;
    int32_t eos = 0;
    int k = -1;
    std::vector<float> logits;
    std::vector<TokenLogprobs> last;
    uint32_t seqLen() const override { return seq; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override {
        std::printf("POS %u %zu\n", pos, tokens.size());
        prefillEnd = pos + (uint32_t)tokens.size();
    }
    int32_t next(int32_t token, uint32_t pos, Sampler &s) override {
        int32_t t = eos;
        if (pos + 1 - prefillEnd <= eosAfter) {
            logits.resize(s.vocabSize());
            for (uint32_t i = 0; i < s.vocabSize(); i++)
                logits[i] = (float)((i * 2654435761u + (uint32_t)token * 97u + pos * 13u) % 1000u) / 100.0f;
            t = s.sample(logits.data());
        }
        if (k >= 0) {
            TokenLogprobs e;
            e.token = t;
            e.logprob = -(float)(pos % 7) * 0.37f;
            for (int j = 0; j < k; j++) e.top.push_back({(int32_t)((t + 31 * j) % vocab), -(float)j * 0.2517f - 0.001f});
            last = {e};
        }
        return t;
    }
    void setLogprobs(int kk) override { k = kk; }
    std::vector<TokenLogprobs> lastLogprobs() override { return last; }
};

int main(int argc, char **argv) {
    if (argc < 4) { std::fprintf(stderr, "usage: api_stop_stub <tokenizer.t> <port> <max-requests> [eos-after]\n"); return 2; }
    Tokenizer tok(argv[1]);
    StopStub b;
    b.vocab = tok.vocabSize();
    b.eos = tok.data().eosIds.at(0);
    if (argc > 4) b.eosAfter = (uint32_t)std::atoi(argv[4]);
    ApiConfig cfg;
    cfg.host = "127.0.0.1";
    cfg.port = std::atoi(argv[2]);
    cfg.maxRequests = std::atoi(argv[3]);
    cfg.temperature = 0.f;
    ApiServer server(b, tok, cfg);
    server.serve();
    std::fflush(stdout);
    return 0;
}
