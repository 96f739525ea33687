// Text stack: `.t` tokenizer file, BPE encoder / streaming decoder, sampler, chat templates, stop detector.
//
// Behavioural parity targets: reference src/tokenizer.cpp:42-164 (file format), :311-390 (encode),
// :224-309 (decode), :405-512 (sampler + xorshift* RNG at :25-36), :522-539 (chat stops),
// :549-637 (templates), :639-724 (EosDetector); converter/tokenizer-writer.py:3-57 (writer).
// The implementation is new: byte strings + hash maps instead of sorted C-string tables, an incremental
// pair-merge loop, std::string based stop detection.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

namespace dl {

constexpr int32_t kTokenizerMagic = 0x567124;
constexpr int32_t kTokenizerMagicOld = 0x567123;

struct TokenizerData {
    std::vector<std::string> vocab;   // raw bytes per token id
    std::vector<float> scores;
    int32_t bosId = -1;
    bool addBos = true;
    std::vector<int32_t> eosIds;
    std::string chatTemplate;         // may be empty
    uint32_t maxTokenLength = 0;
};

TokenizerData readTokenizerFile(const std::string &path);
void writeTokenizerFile(const std::string &path, const TokenizerData &d);

class Tokenizer {
public:
    explicit Tokenizer(const std::string &path);
    explicit Tokenizer(TokenizerData data);

    // addSpecialTokens: match special tokens (id >= bosId) as literal prefixes of the remaining text.
    std::vector<int32_t> encode(const std::string &text, bool isStart, bool addSpecialTokens) const;
    // Streaming decode: returns the longest UTF-8-complete text available after appending `token`.
    // Invalid sequences are replaced by U+FFFD. BOS yields "", EOS flushes whatever is pending.
    std::string decode(int32_t token);
    void resetDecoder() { pending_.clear(); }
    // The same streaming decode with the caller's pending bytes: one state per sequence (the choices of one request).
    std::string decodeWith(std::string &pending, int32_t token) const;
    bool isEos(int32_t token) const;
    std::string describe() const;   // the "📄 ..." lines

    const TokenizerData &data() const { return d_; }
    uint32_t vocabSize() const { return (uint32_t)d_.vocab.size(); }
    uint32_t regularVocabSize() const { return regularSize_; }

private:
    void index();
    int32_t findRegular(const std::string &s) const;
    TokenizerData d_;
    uint32_t regularSize_ = 0;
    std::unordered_map<std::string, int32_t> regular_;
    std::vector<int32_t> specials_;   // ids >= bosId in id order
    std::string pending_;
};

// Seed of choice i of a request for several completions: choice 0 keeps the request's seed (so it draws what a one-completion
// request draws), the others get a splitmix64 mix of (seed, i). The host and device samplers, and both servers, use this.
inline uint64_t choiceSeed(uint64_t seed, uint32_t i) {
    if (i == 0) return seed;
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (uint64_t)i;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// xorshift* generator shared by the host and (by passing the drawn coin) the device sampler.
struct Rng {
    uint64_t state;
    explicit Rng(uint64_t seed) : state(seed) {}
    uint32_t nextU32();
    float nextF32();   // [0, 1)
};

void softmaxInPlace(float *x, size_t n);

// Limits of the sampling controls (presence / frequency penalties and logit bias): both API servers refuse requests beyond them.
// One tensor-parallel control packet carries every bias entry.
constexpr float kMaxPenalty = 2.0f;
constexpr float kMaxLogitBias = 100.0f;
constexpr uint32_t kMaxLogitBiasEntries = 100;

class Sampler {
public:
    Sampler(uint32_t vocabSize, float temperature, float topp, uint64_t seed);
    // Modifies logits in place (controls, temperature, softmax). With controls active, counts the drawn token.
    int32_t sample(float *logits);
    // Sampling controls of the following draws (presence / frequency penalty, logit bias as (id, value) pairs, ids < vocabSize).
    // Before temperature every logit becomes, in float32 without contraction: x = l + bias (if any bias is given), then, for a
    // token this completion has drawn c > 0 times, x = x - c * frequency, then x = x - presence. The device sampler
    // (csrc/cuda/sampler.cu) computes the same numbers. All zero and no bias: off, and sampling is exactly as without controls.
    // Setting the controls starts a new completion (counts from zero, a new completion generation), so device-side copies keyed
    // on the generation always hold the controls in force.
    void setControls(float presence, float frequency, const std::vector<std::pair<int32_t, float>> &bias);
    // Sampling filters of the following temperature > 0 draws (top_k, min_p); they persist until changed. With e[i] =
    // exp(x[i] / T - max(x / T)) from the shared exp, the candidate set S keeps the ids that pass both active filters: top_k the
    // topK first ids in the order (e desc, id asc), min_p those with e[i] >= f32(minP * max e). Ids outside S get e = 0 before
    // the fixed-point normaliser, the nucleus pre-filter divides by |S| - 1, and |S| == 1 returns that id (the coin is drawn
    // all the same). topK 0 (or >= vocabSize) and minP 0 are off. The device sampler computes the same set.
    void setFilters(uint32_t topK, float minP);   // minP in [0, 1]
    uint32_t topK() const { return topK_; }
    float minP() const { return minP_; }
    bool filtersActive() const { return (topK_ > 0 && topK_ < vocabSize_) || minP_ > 0.f; }
    // Starts a completion: zeroes the counts and takes a new completion generation.
    void beginCompletion();
    void applyControls(float *logits) const;   // the transform above, in place ([vocabSize])
    bool controlsActive() const { return presence_ != 0.f || frequency_ != 0.f || !bias_.empty(); }
    float presencePenalty() const { return presence_; }
    float frequencyPenalty() const { return frequency_; }
    const std::vector<std::pair<int32_t, float>> &logitBias() const { return bias_; }
    const std::vector<uint32_t> &counts() const { return counts_; }   // per token of this completion (empty while controls are off)
    // Unique in the process across all samplers: a new sampler and every beginCompletion take a fresh one, so device-side count
    // rows keyed on it are zeroed for every completion, including a fresh sampler per choice.
    uint64_t completionGeneration() const { return completion_; }
    float nextCoin() { return rng_.nextF32(); }
    // A fresh 64-bit seed drawn from this sampler's generator (advances it): the base seed of a request for several
    // completions that names no seed, so that repeated requests differ.
    uint64_t nextSeed() { const uint64_t hi = rng_.nextU32(); return (hi << 32) | rng_.nextU32(); }
    void setTemperature(float t) { temperature_ = t; }
    void setTopp(float p) { topp_ = p; }
    void setSeed(uint64_t s) { rng_.state = s; seed_ = s; seedGeneration_++; }
    uint64_t seed() const { return seed_; }                       // last seed given (constructor or setSeed)
    uint32_t seedGeneration() const { return seedGeneration_; }   // bumped by every setSeed: device-side generators re-seed on change
    float temperature() const { return temperature_; }
    float topp() const { return topp_; }
    uint32_t vocabSize() const { return vocabSize_; }

private:
    int32_t draw(float *logits);            // greedy / temperature / top-p draw
    uint32_t applyFilters(float *e);        // zeroes e outside S, returns |S|
    uint32_t vocabSize_;
    uint32_t topK_ = 0;
    float minP_ = 0.f;
    std::vector<float> keys_;
    float temperature_, topp_;
    Rng rng_;
    uint64_t seed_ = 0;
    uint32_t seedGeneration_ = 0;
    std::vector<std::pair<float, int32_t>> candidates_;
    float presence_ = 0.f, frequency_ = 0.f;
    std::vector<std::pair<int32_t, float>> bias_;
    std::vector<float> biasDense_;
    std::vector<uint32_t> counts_;
    uint64_t completion_;
};

enum ChatTemplateType : int32_t { TEMPLATE_UNKNOWN = 0, TEMPLATE_LLAMA2 = 1, TEMPLATE_LLAMA3 = 2, TEMPLATE_DEEP_SEEK3 = 3, TEMPLATE_CHATML = 4 };
ChatTemplateType parseChatTemplateType(const std::string &name);   // "llama2" | "llama3" | "deepSeek3" | "chatml"
const char *chatTemplateTypeName(ChatTemplateType t);

struct ChatItem { std::string role, message; };
struct GeneratedChat { std::string content; std::string publicPrompt; };

class ChatTemplateGenerator {
public:
    ChatTemplateGenerator(ChatTemplateType type, const std::string &chatTemplate, const std::string &eos);
    GeneratedChat generate(const std::vector<ChatItem> &items, bool appendGenerationPrompt) const;
    ChatTemplateType type() const { return type_; }
private:
    ChatTemplateType type_;
    std::string eos_;
};

enum EosDetectorResult : int32_t { MAYBE_EOS = 0, EOS = 1, NOT_EOS = 2 };

// Streaming stop detector. Pieces are appended; a stop string may appear after up to `paddingLeft`
// leading bytes and be followed by up to `paddingRight` bytes inside the buffered text.
class EosDetector {
public:
    EosDetector(std::vector<int32_t> tokens, std::vector<std::string> pieces, int paddingLeft, int paddingRight);
    EosDetectorResult append(int32_t tokenId, const std::string &piece);
    bool isEos(int32_t tokenId) const;
    // Text that may be shown to the user; empty when nothing (or only the stop) is buffered.
    std::string getDelta() const;
    void reset();
private:
    std::vector<int32_t> tokens_;
    std::vector<std::string> pieces_;
    int padLeft_, padRight_;
    std::string buffer_;
    int eosPos_ = -1;
};

// Limits of a request's `stop` strings (both API servers refuse requests beyond them): they bound the bytes a StopMatcher holds
// back and its work per token.
constexpr size_t kMaxStopStrings = 4;
constexpr size_t kMaxStopBytes = 256;

// A completion's `stop` strings, matched on the bytes of its generated text G (the concatenation of the deltas an EosDetector
// releases). push() takes the next delta and returns the bytes that can no longer be cut: it holds back the longest suffix of the
// text not yet returned that is a proper prefix of some stop string. At the first delta that completes an occurrence of any stop
// string, it returns G up to the start of the earliest-starting occurrence (minus what it returned before) and stopped() turns
// true; the stop string and everything after it are never returned. flush() returns the held bytes at any other end.
class StopMatcher {
public:
    explicit StopMatcher(std::vector<std::string> stops);   // every string non-empty
    std::string push(const std::string &delta);
    std::string flush();
    bool stopped() const { return stopped_; }
    const std::string &held() const { return held_; }
private:
    std::vector<std::string> stops_;
    std::string held_;
    bool stopped_ = false;
};

}  // namespace dl
