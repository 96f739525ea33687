// CPU-only harness for `logprobs` in csrc/app/api_server.cpp: the real HTTP / JSON / validation code over a fake model whose logits
// are a fixed function of (token, position, vocabulary id), drawn by the host Sampler, and whose log-probability entries are a
// fixed float32 function of (drawn token, position, k). tests/test_logprobs_args.py runs its Python twin through the Python server.
// With a third argument "tp" the backend refuses logprobs like a tensor-parallel job.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

struct LogprobsStub : InferenceBackend {
    uint32_t vocab = 0, seq = 4096, eosAfter = 12, prefillEnd = 0;
    int32_t eos = 0;
    int k = -1;
    bool tp = false;
    std::vector<float> logits;
    std::vector<TokenLogprobs> last;
    uint32_t seqLen() const override { return seq; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) override { prefillEnd = pos + (uint32_t)tokens.size(); }
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
    void setLogprobs(int kk) override {
        if (kk >= 0 && tp) throw std::runtime_error("logprobs are not supported under tensor parallelism yet");
        k = kk;
    }
    std::vector<TokenLogprobs> lastLogprobs() override { return last; }
};

int main(int argc, char **argv) {
    if (argc < 4) { std::fprintf(stderr, "usage: api_logprobs_stub <tokenizer.t> <port> <max-requests> [tp]\n"); return 2; }
    Tokenizer tok(argv[1]);
    LogprobsStub b;
    b.vocab = tok.vocabSize();
    b.eos = tok.data().eosIds.at(0);
    b.tp = argc > 4 && std::string(argv[4]) == "tp";
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
