// Native `dllama-api`: blocking HTTP/1.1 server with the reference's routes (src/dllama-api.cpp:43-632, src/api-types.hpp):
//   POST /v1/chat/completions (JSON body; JSON response or SSE-style chunked stream), GET /v1/models, OPTIONS * (CORS), else 404.
// One request at a time over one KV sequence with NaiveCache prefix re-use. The inference side is an interface so the HTTP /
// JSON / template / stop-detector plumbing can be exercised without a GPU (tests/native/api_choices_stub_main.cpp).
#pragma once
#include <cstdint>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "../host/text.hpp"
#include "json.hpp"

namespace dl {

constexpr int kMaxTopLogprobs = 20;   // the largest `top_logprobs` (csrc/cuda/logprobs.cu)

// The log-probabilities of one drawn token: its logprob and the k most likely (id, logprob) in the order (logprob desc, id asc).
struct TokenLogprobs {
    int32_t token = -1;
    float logprob = 0.f;
    std::vector<std::pair<int32_t, float>> top;
};

struct InferenceBackend {
    virtual ~InferenceBackend() {}
    virtual uint32_t seqLen() const = 0;
    virtual uint32_t vocabSize() const = 0;
    virtual void setVocabLimit(uint32_t) {}   // greedy decoding never returns ids >= limit (tokenizer vocabulary)
    virtual void prefill(const std::vector<int32_t> &tokens, uint32_t pos) = 0;
    virtual int32_t next(int32_t token, uint32_t pos, Sampler &sampler) = 0;   // greedy on the device when temperature == 0
    // Greedy speculative decoding with a draft model (--draft-model): whether a single completion with the sampler's settings
    // decodes in rounds (plain greedy only), and one round from the last emitted token at `pos`: the tokens greedy decoding emits next.
    virtual bool speculates(const Sampler & /*sampler*/) const { return false; }
    virtual std::vector<int32_t> specRound(int32_t /*token*/, uint32_t /*pos*/) { throw std::runtime_error("no draft model"); }
    // Several completions of one prompt (runChoices). Without a batched path the choices run one after another through next().
    virtual bool batchedChoices(uint32_t /*n*/) const { return false; }
    virtual void seedChoices(const std::vector<uint64_t> & /*seeds*/) {}
    // the sampler's controls for the batched choices, each choice's counts from zero
    virtual void choiceControls(const Sampler & /*sampler*/, uint32_t /*n*/) {}
    // first tokens of n choices, all drawn from the logits of `token` at P
    virtual std::vector<int32_t> choicesFirst(int32_t /*token*/, uint32_t /*P*/, uint32_t /*n*/, float /*temperature*/, float /*topp*/) { return {}; }
    // one batched step: choice b feeds tokens[b] at rotary position P + 1 + j, cache row P + 1 + b * C + j (active choices only)
    virtual std::vector<int32_t> choicesStep(const std::vector<int32_t> & /*tokens*/, uint32_t /*P*/, uint32_t /*C*/, uint32_t /*j*/,
                                             uint32_t /*activeMask*/, float /*temperature*/, float /*topp*/) { return {}; }
    // the sequential path re-seeds the single-sequence generator per choice; these keep its stream across the request
    virtual uint64_t saveSampler() { return 0; }
    virtual void restoreSampler(uint64_t /*saved*/) {}
    // KV-cache slots (--parallel): independent sequences decoded together, one batched step per token. slots() == 0: unsupported.
    virtual uint32_t slots() const { return 0; }
    virtual uint32_t slotLen() const { return 0; }
    virtual void slotPrefill(uint32_t /*slot*/, const std::vector<int32_t> & /*tokens*/, uint32_t /*pos*/) { throw std::runtime_error("slots unsupported"); }
    virtual void slotCopy(uint32_t /*src*/, uint32_t /*dst*/, uint32_t /*P*/) { throw std::runtime_error("slots unsupported"); }
    // Paged slots (paged() true: the slots share the cache as one pool of 64-row pages, csrc/cuda/engine.cu): slotReserve grows a slot
    // to cover rows [0, rows) (false, nothing changed, when the pool is short), slotTrim keeps the pages of rows [0, rows) and frees
    // the rest, slotRelease frees every page of a slot; freePages and slotPageCount report the pool.
    virtual bool paged() const { return false; }
    virtual bool slotReserve(uint32_t /*slot*/, uint32_t /*rows*/) { throw std::runtime_error("paged slots unsupported"); }
    virtual void slotTrim(uint32_t /*slot*/, uint32_t /*rows*/) { throw std::runtime_error("paged slots unsupported"); }
    virtual void slotRelease(uint32_t /*slot*/) { throw std::runtime_error("paged slots unsupported"); }
    virtual uint32_t freePages() const { return 0; }
    virtual uint32_t slotPageCount(uint32_t /*slot*/) const { return 0; }
    // seeds slot `slot`'s generator, zeroes its counts and sets its temperature (0: arg-max), top-p, penalties and logit bias
    virtual void slotSampling(uint32_t /*slot*/, uint64_t /*seed*/, float /*temperature*/, float /*topp*/, float /*presence*/, float /*frequency*/,
                              const std::vector<std::pair<int32_t, float>> & /*bias*/) { throw std::runtime_error("slots unsupported"); }
    // slot `slot`'s top_k / min_p (Sampler::setFilters), called after slotSampling (which switches them off) only when one is on
    virtual void slotFilters(uint32_t /*slot*/, uint32_t /*topK*/, float /*minP*/) { throw std::runtime_error("sampling filters unsupported"); }
    // row b feeds tokens[b] at pos[b] of slot b (active rows: bit b of activeMask); returns each active row's draw
    virtual std::vector<int32_t> slotsStep(const std::vector<int32_t> & /*tokens*/, const std::vector<int32_t> & /*pos*/, uint32_t /*activeMask*/) {
        throw std::runtime_error("slots unsupported");
    }
    // Log-probabilities of the following next / choicesFirst / choicesStep draws with k (0..20) top entries, -1: none (throws where
    // they cannot run, e.g. under tensor parallelism). lastLogprobs(): one entry per row of the last such call.
    virtual void setLogprobs(int k) { if (k >= 0) throw std::runtime_error("logprobs are not supported by this backend"); }
    virtual std::vector<TokenLogprobs> lastLogprobs() { return {}; }
    // slot `slot`'s draws with k top entries (-1: none; every slotSampling resets it), and slotsStep that also returns them
    virtual void slotLogprobs(uint32_t /*slot*/, int k) { if (k >= 0) throw std::runtime_error("logprobs are not supported by this backend"); }
    virtual std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> & /*tokens*/, const std::vector<int32_t> & /*pos*/,
                                                   uint32_t /*activeMask*/, std::vector<TokenLogprobs> & /*rows*/) {
        throw std::runtime_error("logprobs are not supported by this backend");
    }
};

// One row's result block of the log-probability kernel (kApiLogprobsWords int32 words, csrc/cuda/engine_api.h) decoded.
TokenLogprobs decodeLogprobs(const int32_t *words);

constexpr uint32_t kMaxChoices = 8;   // the engine's widest batch: one row per choice

// n completions of the prompt whose last token `token` sits at P (everything before it prefilled); choice i draws with
// choiceSeed(baseSeed, i), its j-th token has rotary position P + 1 + j and cache row P + 1 + i * C + j with
// C = (seqLen - 1 - P) / n, and it stops after min(maxTokens, C) tokens (maxTokens <= 0: C). A single completion (n = 1) is the
// single-sequence loop of the CLIs instead: it stops after min(maxTokens, seqLen - P) tokens, so it may fill the context up to
// its last row. onToken(i, token) returns true when choice i is finished. The sampler's controls apply to every choice, each with
// its own counts from zero, and so do its filters (top_k / min_p; choiceControls hands them to the batched path). Same rules as distributed_llama_b200.api.run_choices.
// onLogprobs (optional, with backend.setLogprobs(k) made): called with each token's entry right before onToken(i, token).
std::vector<std::vector<int32_t>> runChoices(InferenceBackend &backend, int32_t token, uint32_t P, uint32_t n, int maxTokens, uint32_t seqLen,
                                             Sampler &sampler, uint64_t baseSeed, const std::function<bool(uint32_t, int32_t)> &onToken,
                                             const std::function<void(uint32_t, const TokenLogprobs &)> &onLogprobs = nullptr);

struct HttpRequest {
    int fd = -1;
    std::string method = "UNKNOWN", path, body;
    std::map<std::string, std::string> headers;   // lower-cased names
    JsonValue json;
    bool hasJson = false;

    static HttpRequest read(int fd);   // throws std::runtime_error on socket / protocol errors
    void writeCors() const;
    void writeNotFound() const;
    void writeJson(const std::string &text) const;
    void writeStreamStart() const;
    void writeStreamChunk(const std::string &data) const;
    void writeStreamEnd() const;
private:
    void send(const std::string &data) const;
};

// (endPos, message) per chat turn; re-used only if *all* cached messages are an exact prefix of the new history.
class NaiveCache {
public:
    void push(uint32_t endPos, const ChatItem &msg) { items_.push_back({endPos, msg}); }
    void clear() { items_.clear(); }
    size_t size() const { return items_.size(); }
    // Returns the position generation restarts from and trims `messages` to the part that still has to be evaluated.
    uint32_t resolveDeltaPrompt(std::vector<ChatItem> &messages);
    // How many cached messages resolveDeltaPrompt would re-use for `messages` (0: none).
    size_t coveredPrefix(const std::vector<ChatItem> &messages) const;
    void copyFrom(const NaiveCache &o) { items_ = o.items_; }
private:
    struct Item { uint32_t endPos; ChatItem msg; };
    std::vector<Item> items_;
};

// one streamed `chat.completion` chunk; `logprobs` (entries as JSON text, may be empty) adds "logprobs": {"content": [...]}
std::string chunkJson(const std::string *delta, bool stop, uint32_t index = 0, const std::vector<std::string> *logprobs = nullptr);

// The request's log-probabilities: -1 without them, else the number of top entries; the rules of
// distributed_llama_b200.apps.api_server.parse_logprobs (throws on anything else).
int parseLogprobs(const JsonValue &body);
// The request's `stop` strings (none when absent, null or []): a string or an array of at most kMaxStopStrings strings, each 1 to
// kMaxStopBytes bytes of UTF-8 after unescaping, without unpaired surrogate escapes. The rules of
// distributed_llama_b200.apps.api_server.parse_stop (throws on anything else).
std::vector<std::string> parseStop(const JsonValue &body);
// One token's response entry {"token", "logprob", "bytes", "top_logprobs"}, formatted as the Python server's json.dumps does.
std::string logprobEntryJson(const Tokenizer &tok, const TokenLogprobs &e);

// A --presence-penalty / --frequency-penalty value: a number in [-kMaxPenalty, kMaxPenalty] (throws otherwise).
float parsePenalty(const std::string &flag, const std::string &value);
// The request's sampling filters: `top_k` an integer from 0 to kMaxTopK, `min_p` a number from 0 to 1; absent fields keep the
// values passed in (the server's defaults). The rules of distributed_llama_b200.apps.api_server.parse_filters (throws otherwise).
constexpr uint32_t kMaxTopK = 2147483647u;
void parseFilters(const JsonValue &body, uint32_t &topK, float &minP);
// --top-k / --min-p values, in the ranges above (throws otherwise).
uint32_t parseTopK(const std::string &flag, const std::string &value);
float parseMinP(const std::string &flag, const std::string &value);

struct ApiConfig {
    std::string host = "0.0.0.0", modelName = "model", chatTemplate;
    int port = 9990;
    float temperature = 0.8f, topp = 0.9f;
    float presencePenalty = 0.f, frequencyPenalty = 0.f;   // defaults of the request fields
    uint32_t topK = 0;
    float minP = 0.f;
    uint64_t seed = 0;
    int maxRequests = 0;   // 0 = serve forever
    uint32_t parallel = 1; // > 1: that many requests decoded together in KV-cache slots (serveParallel)
};

class ApiServer {
public:
    ApiServer(InferenceBackend &backend, Tokenizer &tokenizer, const ApiConfig &cfg);
    void complete(HttpRequest &req);
    void models(HttpRequest &req) const;
    void serve();          // accept loop (parallel > 1: serveParallel)
private:
    void serveParallel(int srv);   // one engine thread running SlotScheduler (host/slot_scheduler.hpp), a reader thread per connection
    InferenceBackend &backend_;
    Tokenizer &tok_;
    ApiConfig cfg_;
    Sampler sampler_;
    NaiveCache cache_;
    std::vector<std::string> stops_;
    ChatTemplateGenerator gen_;
};

}  // namespace dl
