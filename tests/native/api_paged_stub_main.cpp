// CPU-only harness for the --parallel server of csrc/app/api_server.cpp over paged KV-cache slots: the real HTTP / JSON / template /
// per-slot NaiveCache / scheduling code over a fake slot backend whose slots share a pool of 64-row pages, kept the way the engine
// keeps them (csrc/cuda/engine.cu: lowest free page first). A row's next token is a fixed function of (token, position, and its
// slot's seed when sampling); EOS comes after `eos-after` tokens of a completion. A step that feeds a row outside its slot's pages
// exits with status 3. The Python twin is PagedSlotStub in tests/test_paged_slots_servers.py.
// Prints "POS <slot> <start> <n>" for every prefill and "FREE <slot>" for every slot whose pages go back to the pool.
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../csrc/app/api_server.hpp"

using namespace dl;

constexpr uint32_t kPage = 64;

struct PagedSlotStub : InferenceBackend {
    uint32_t vocab = 0, regular = 0, n = 2, pages = 4, eosAfter = 10;
    int32_t eos = 0;
    std::vector<uint64_t> seed;
    std::vector<float> temp;
    std::vector<uint32_t> produced;
    std::vector<std::vector<uint32_t>> table;
    std::vector<bool> used;
    uint32_t seqLen() const override { return pages * kPage; }
    uint32_t vocabSize() const override { return vocab; }
    void prefill(const std::vector<int32_t> &, uint32_t) override { throw std::runtime_error("single-sequence call in --parallel mode"); }
    int32_t next(int32_t, uint32_t, Sampler &) override { throw std::runtime_error("single-sequence call in --parallel mode"); }
    uint32_t slots() const override { return n; }
    uint32_t slotLen() const override { return pages * kPage; }
    bool paged() const override { return true; }
    bool slotReserve(uint32_t slot, uint32_t rows) override {
        const uint32_t want = (rows + kPage - 1) / kPage;
        if (want <= table[slot].size()) return true;
        uint32_t nFree = 0;
        for (bool u : used) nFree += u ? 0 : 1;
        if (nFree < want - table[slot].size()) return false;
        for (uint32_t p = 0; p < pages && table[slot].size() < want; p++)
            if (!used[p]) { used[p] = true; table[slot].push_back(p); }
        return true;
    }
    void slotTrim(uint32_t slot, uint32_t rows) override {
        const uint32_t keep = (rows + kPage - 1) / kPage;
        while (table[slot].size() > keep) { used[table[slot].back()] = false; table[slot].pop_back(); }
    }
    void slotRelease(uint32_t slot) override {
        if (!table[slot].empty()) std::printf("FREE %u\n", slot);
        slotTrim(slot, 0);
    }
    uint32_t freePages() const override {
        uint32_t nFree = 0;
        for (bool u : used) nFree += u ? 0 : 1;
        return nFree;
    }
    uint32_t slotPageCount(uint32_t slot) const override { return (uint32_t)table[slot].size(); }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) override {
        if (pos + tokens.size() > table[slot].size() * kPage) std::exit(3);
        std::printf("POS %u %u %zu\n", slot, pos, tokens.size());
    }
    void slotCopy(uint32_t, uint32_t dst, uint32_t P) override {
        if (!slotReserve(dst, P)) std::exit(3);
    }
    void slotSampling(uint32_t slot, uint64_t s, float temperature, float, float, float, const std::vector<std::pair<int32_t, float>> &) override {
        seed[slot] = s;
        temp[slot] = temperature;
        produced[slot] = 0;
    }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask) override {
        std::vector<int32_t> out(n, -1);
        for (uint32_t b = 0; b < n; b++) {
            if (!((activeMask >> b) & 1u)) continue;
            if ((uint32_t)pos[b] >= table[b].size() * kPage) std::exit(3);
            const uint64_t salt = temp[b] > 0.f ? (seed[b] % 997u) * 31u : 0u;
            out[b] = ++produced[b] > eosAfter ? eos : (int32_t)(((uint64_t)tokens[b] * 7u + (uint64_t)pos[b] * 13u + 5u + salt) % regular);
        }
        return out;
    }
};

int main(int argc, char **argv) {
    if (argc < 7) {
        std::fprintf(stderr, "usage: api_paged_stub <tokenizer.t> <port> <max-requests> <parallel> <pages> <eos-after>\n");
        return 2;
    }
    Tokenizer tok(argv[1]);
    PagedSlotStub b;
    b.vocab = tok.vocabSize();
    b.regular = tok.regularVocabSize();
    b.eos = tok.data().eosIds.at(0);
    b.n = (uint32_t)std::atoi(argv[4]);
    b.pages = (uint32_t)std::atoi(argv[5]);
    b.eosAfter = (uint32_t)std::atoi(argv[6]);
    b.seed.assign(b.n, 0);
    b.temp.assign(b.n, 0.f);
    b.produced.assign(b.n, 0);
    b.table.assign(b.n, {});
    b.used.assign(b.pages, false);
    ApiConfig cfg;
    cfg.host = "127.0.0.1";
    cfg.port = std::atoi(argv[2]);
    cfg.maxRequests = std::atoi(argv[3]);
    cfg.modelName = "stub.m";
    cfg.temperature = 0.f;
    cfg.seed = 77;
    cfg.parallel = b.n;
    ApiServer server(b, tok, cfg);
    server.serve();
    return 0;
}
