#include "text.hpp"

#include "../common/dl_expf.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <functional>
#include <stdexcept>

namespace dl {

// ---- .t file -----------------------------------------------------------------------------------

namespace {
enum TokKey : int32_t {
    TK_VERSION = 0, TK_VOCAB_SIZE = 1, TK_MAX_TOKEN_LENGTH = 2, TK_BOS_ID = 3, TK_EOS_ID = 4, TK_PAD_ID = 5,
    TK_CHAT_EOS_ID = 6, TK_CHAT_TEMPLATE = 7, TK_CHAT_STOP = 8, TK_N_EOS_TOKENS = 9, TK_ADD_BOS = 10,
};

template <typename T> T readPod(std::ifstream &f, const char *what) {
    T v;
    f.read(reinterpret_cast<char *>(&v), sizeof(T));
    if (!f) throw std::runtime_error(std::string("Cannot read ") + what + " from tokenizer file");
    return v;
}
template <typename T> void writePod(std::ofstream &f, T v) { f.write(reinterpret_cast<const char *>(&v), sizeof(T)); }
}  // namespace

TokenizerData readTokenizerFile(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("Failed to open tokenizer file");
    TokenizerData d;
    uint32_t vocabSize = 0;
    const int32_t magic = readPod<int32_t>(f, "magic");
    if (magic == kTokenizerMagicOld) {
        vocabSize = readPod<uint32_t>(f, "header");
        d.maxTokenLength = readPod<uint32_t>(f, "header");
        d.bosId = readPod<int32_t>(f, "header");
        d.eosIds.push_back(readPod<int32_t>(f, "header"));
        (void)readPod<int32_t>(f, "header");  // pad id
    } else if (magic == kTokenizerMagic) {
        const int32_t headerSize = readPod<int32_t>(f, "header size");
        if (headerSize < 8 || (headerSize - 8) % 8) throw std::runtime_error("Invalid tokenizer header size");
        int32_t version = -1, templateLen = -1, nEos = 0;
        int64_t chatStopSkip = 0;   // legacy key: bytes of an (ignored) stop string stored right after the header
        for (int i = 0; i < (headerSize - 8) / 8; i++) {
            const int32_t key = readPod<int32_t>(f, "header key");
            const int32_t value = readPod<int32_t>(f, "header value");
            switch (key) {
                case TK_VERSION: version = value; break;
                case TK_VOCAB_SIZE: vocabSize = (uint32_t)value; break;
                case TK_MAX_TOKEN_LENGTH: d.maxTokenLength = (uint32_t)value; break;
                case TK_BOS_ID: d.bosId = value; break;
                case TK_EOS_ID: case TK_CHAT_EOS_ID: d.eosIds.push_back(value); break;  // legacy keys
                case TK_CHAT_TEMPLATE: templateLen = value; break;
                case TK_CHAT_STOP: chatStopSkip += value; break;   // applied after the whole header has been read (reference src/tokenizer.cpp:68-86)
                case TK_PAD_ID: break;
                case TK_N_EOS_TOKENS: nEos = value; break;
                case TK_ADD_BOS: d.addBos = value == 1; break;
                default: throw std::runtime_error("Invalid tokenizer header key:" + std::to_string(key));
            }
        }
        if (version != 1) throw std::runtime_error("Old tokenizer version, please regenerate your tokenizer");
        if (chatStopSkip > 0) f.seekg(chatStopSkip, std::ios::cur);
        if (templateLen > 0) {
            d.chatTemplate.resize(templateLen);
            f.read(&d.chatTemplate[0], templateLen);
            if (!f) throw std::runtime_error("Cannot read chat template from tokenizer file");
        }
        for (int i = 0; i < nEos; i++) d.eosIds.push_back(readPod<int32_t>(f, "eos token id"));
    } else {
        throw std::runtime_error("Invalid tokenizer file");
    }
    if (d.maxTokenLength < 1) throw std::runtime_error("Invalid tokenizer max token length");
    d.vocab.resize(vocabSize);
    d.scores.resize(vocabSize);
    for (uint32_t i = 0; i < vocabSize; i++) {
        d.scores[i] = readPod<float>(f, "score");
        const int32_t len = readPod<int32_t>(f, "length");
        if (len < 0 || len > (1 << 20)) throw std::runtime_error("Cannot read word from tokenizer file");
        d.vocab[i].resize(len);
        if (len) f.read(&d.vocab[i][0], len);
        if (!f) throw std::runtime_error("Cannot read word from tokenizer file");
    }
    return d;
}

void writeTokenizerFile(const std::string &path, const TokenizerData &d) {
    std::ofstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("Cannot create tokenizer file");
    uint32_t maxLen = 0;
    for (const auto &t : d.vocab) maxLen = std::max<uint32_t>(maxLen, (uint32_t)t.size());
    std::vector<std::pair<int32_t, int32_t>> kv;
    kv.push_back({TK_BOS_ID, d.bosId});
    kv.push_back({TK_VERSION, 1});
    kv.push_back({TK_VOCAB_SIZE, (int32_t)d.vocab.size()});
    kv.push_back({TK_MAX_TOKEN_LENGTH, (int32_t)maxLen});
    if (!d.chatTemplate.empty()) kv.push_back({TK_CHAT_TEMPLATE, (int32_t)d.chatTemplate.size()});
    kv.push_back({TK_N_EOS_TOKENS, (int32_t)d.eosIds.size()});
    kv.push_back({TK_ADD_BOS, d.addBos ? 1 : 0});
    writePod<int32_t>(f, kTokenizerMagic);
    writePod<int32_t>(f, (int32_t)(8 + 8 * kv.size()));
    for (auto &p : kv) { writePod<int32_t>(f, p.first); writePod<int32_t>(f, p.second); }
    f.write(d.chatTemplate.data(), d.chatTemplate.size());
    for (int32_t e : d.eosIds) writePod<int32_t>(f, e);
    for (size_t i = 0; i < d.vocab.size(); i++) {
        if (d.vocab[i].empty()) throw std::runtime_error("Empty token in vocabulary");
        writePod<float>(f, d.scores[i]);
        writePod<uint32_t>(f, (uint32_t)d.vocab[i].size());
        f.write(d.vocab[i].data(), d.vocab[i].size());
    }
}

// ---- Tokenizer -----------------------------------------------------------------------------------

Tokenizer::Tokenizer(const std::string &path) : d_(readTokenizerFile(path)) { index(); }
Tokenizer::Tokenizer(TokenizerData data) : d_(std::move(data)) { index(); }

void Tokenizer::index() {
    // The format has no explicit "special token" flag: ids below bosId are regular (mergeable) tokens,
    // ids from bosId upwards are specials that only ever match literally.
    const uint32_t n = (uint32_t)d_.vocab.size();
    regularSize_ = d_.bosId >= 0 ? std::min<uint32_t>((uint32_t)d_.bosId, n) : n;
    regular_.reserve(regularSize_ * 2);
    for (uint32_t i = 0; i < regularSize_; i++) regular_.emplace(d_.vocab[i], (int32_t)i);  // first id wins
    for (uint32_t i = regularSize_; i < n; i++) specials_.push_back((int32_t)i);
    if (d_.maxTokenLength == 0)
        for (auto &t : d_.vocab) d_.maxTokenLength = std::max<uint32_t>(d_.maxTokenLength, (uint32_t)t.size());
}

int32_t Tokenizer::findRegular(const std::string &s) const {
    auto it = regular_.find(s);
    return it == regular_.end() ? -1 : it->second;
}

bool Tokenizer::isEos(int32_t token) const {
    return std::find(d_.eosIds.begin(), d_.eosIds.end(), token) != d_.eosIds.end();
}

std::string Tokenizer::describe() const {
    std::string s;
    if (d_.bosId >= 0) {
        s += "📄 AddBos: " + std::to_string(d_.addBos ? 1 : 0) + "\n";
        s += "📄 BosId: " + std::to_string(d_.bosId) + " (" + d_.vocab[d_.bosId] + ")\n";
    }
    if (!d_.eosIds.empty()) {
        s += "📄 EosId: ";
        for (int32_t e : d_.eosIds) s += std::to_string(e) + " (" + d_.vocab[e] + ") ";
        s += "\n";
    }
    s += "📄 RegularVocabSize: " + std::to_string(regularSize_) + "\n";
    s += "📄 SpecialVocabSize: " + std::to_string(d_.vocab.size() - regularSize_) + "\n";
    return s;
}

std::vector<int32_t> Tokenizer::encode(const std::string &text, bool isStart, bool addSpecialTokens) const {
    std::vector<int32_t> toks;
    toks.reserve(text.size() + 1);
    if (isStart && d_.addBos && d_.bosId >= 0) toks.push_back(d_.bosId);

    // Pass 1: greedy segmentation into known regular tokens (shortest prefix that is a token), with
    // special tokens matched literally.
    std::string buf;
    for (size_t i = 0; i < text.size();) {
        if (addSpecialTokens) {
            int32_t hit = -1;
            for (int32_t id : specials_) {
                const std::string &v = d_.vocab[id];
                if (!v.empty() && text.compare(i, v.size(), v) == 0) { hit = id; break; }
            }
            if (hit >= 0) {
                toks.push_back(hit);
                i += d_.vocab[hit].size();
                continue;
            }
        }
        buf.push_back(text[i++]);
        const int32_t id = findRegular(buf);
        if (id >= 0) { toks.push_back(id); buf.clear(); }
        else if (buf.size() > d_.maxTokenLength) throw std::runtime_error("Tokenizer: cannot segment input text");
    }
    if (!buf.empty()) throw std::runtime_error("Tokenizer: trailing bytes cannot be tokenized");

    // Pass 2: repeatedly merge the adjacent pair whose concatenation is a regular token with the highest
    // score (leftmost on ties). Only the two pairs touching a merge site are re-evaluated.
    auto pairId = [&](size_t i) -> int32_t {
        std::string cat = d_.vocab[toks[i]];
        cat += d_.vocab[toks[i + 1]];
        return findRegular(cat);
    };
    std::vector<int32_t> cand(toks.size() > 0 ? toks.size() - 1 : 0);
    for (size_t i = 0; i + 1 < toks.size(); i++) cand[i] = pairId(i);
    for (;;) {
        float best = -1e10f;
        int bestIdx = -1;
        for (size_t i = 0; i < cand.size(); i++)
            if (cand[i] >= 0 && d_.scores[cand[i]] > best) { best = d_.scores[cand[i]]; bestIdx = (int)i; }
        if (bestIdx < 0) break;
        toks[bestIdx] = cand[bestIdx];
        toks.erase(toks.begin() + bestIdx + 1);
        cand.erase(cand.begin() + bestIdx);
        if (bestIdx > 0) cand[bestIdx - 1] = pairId(bestIdx - 1);
        if ((size_t)bestIdx < cand.size()) cand[bestIdx] = pairId(bestIdx);
    }
    return toks;
}

std::string Tokenizer::decodeWith(std::string &pending, int32_t token) const {
    if (token == d_.bosId) return std::string();
    if (isEos(token)) {
        std::string rest;
        rest.swap(pending);
        return rest;
    }
    if (token < 0 || (size_t)token >= d_.vocab.size()) throw std::runtime_error("Tokenizer: token id out of range");
    pending += d_.vocab[token];

    static const char kReplacement[] = "\xEF\xBF\xBD";
    std::string out;
    size_t i = 0, committed = 0;   // bytes [0, committed) of pending are fully consumed
    const size_t n = pending.size();
    while (i < n) {
        const unsigned char c = (unsigned char)pending[i];
        size_t need;
        if (c <= 0x7f) need = 0;
        else if (c >= 0xc0 && c <= 0xdf) need = 1;
        else if (c >= 0xe0 && c <= 0xef) need = 2;
        else if (c >= 0xf0 && c <= 0xf7) need = 3;
        else { out += kReplacement; i++; committed = i; continue; }   // stray continuation / invalid lead
        size_t have = 0;
        while (have < need && i + 1 + have < n && (((unsigned char)pending[i + 1 + have]) & 0xc0) == 0x80) have++;
        if (have == need) {
            out.append(pending, i, need + 1);
            i += need + 1;
            committed = i;
        } else if (i + 1 + have < n) {
            // sequence interrupted by a non-continuation byte: drop it, resume at the interrupting byte
            out += kReplacement;
            i += 1 + have;
            committed = i;
        } else {
            break;   // incomplete tail: wait for more bytes
        }
    }
    pending.erase(0, committed);
    return out;
}

std::string Tokenizer::decode(int32_t token) { return decodeWith(pending_, token); }

// ---- RNG / sampler ---------------------------------------------------------------------------------

uint32_t Rng::nextU32() {
    state ^= state >> 12;
    state ^= state << 25;
    state ^= state >> 27;
    return (uint32_t)((state * 0x2545F4914F6CDD1Dull) >> 32);
}

float Rng::nextF32() { return (float)(nextU32() >> 8) / 16777216.0f; }

void softmaxInPlace(float *x, size_t n) {
    if (n == 0) return;
    float m = x[0];
    for (size_t i = 1; i < n; i++) m = std::max(m, x[i]);
    float sum = 0.f;
    for (size_t i = 0; i < n; i++) { x[i] = std::exp(x[i] - m); sum += x[i]; }
    const float inv = 1.f / sum;
    for (size_t i = 0; i < n; i++) x[i] *= inv;
}

static uint64_t nextCompletionGeneration() {
    static std::atomic<uint64_t> next{1};
    return next.fetch_add(1);
}

Sampler::Sampler(uint32_t vocabSize, float temperature, float topp, uint64_t seed)
    : vocabSize_(vocabSize), temperature_(temperature), topp_(topp), rng_(seed), seed_(seed), completion_(nextCompletionGeneration()) {}

void Sampler::setControls(float presence, float frequency, const std::vector<std::pair<int32_t, float>> &bias) {
    for (const auto &b : bias)
        if (b.first < 0 || (uint32_t)b.first >= vocabSize_) throw std::invalid_argument("logit_bias: token id outside the vocabulary");
    presence_ = presence;
    frequency_ = frequency;
    bias_ = bias;
    biasDense_.clear();
    if (!bias_.empty()) {
        biasDense_.assign(vocabSize_, 0.f);
        for (const auto &b : bias_) biasDense_[b.first] = b.second;
    }
    if (!controlsActive()) counts_.clear();
    else counts_.assign(vocabSize_, 0u);
    completion_ = nextCompletionGeneration();
}

void Sampler::setFilters(uint32_t topK, float minP) {
    if (!(minP >= 0.f && minP <= 1.f)) throw std::invalid_argument("min_p must lie in [0, 1]");
    topK_ = topK;
    minP_ = minP;
}

// Without FMA, like applyControls: the min_p threshold is one rounded multiply, as the device's __fmul_rn.
uint32_t Sampler::applyFilters(float *e) {
    const uint32_t n = vocabSize_;
    uint32_t kept = n;
    if (minP_ > 0.f) {
        float eMax = 0.f;
        for (uint32_t i = 0; i < n; i++) eMax = std::max(eMax, e[i]);
        const float thr = minP_ * eMax;
        kept = 0;
        for (uint32_t i = 0; i < n; i++) {
            if (e[i] < thr) e[i] = 0.f;
            else kept++;
        }
    }
    if (topK_ > 0 && topK_ < kept) {
        // the K-th value of the order (e desc, id asc); every id above it stays, and the lowest ids among its ties up to K in all
        keys_.assign(e, e + n);
        std::nth_element(keys_.begin(), keys_.begin() + (topK_ - 1), keys_.end(), std::greater<float>());
        const float kth = keys_[topK_ - 1];
        uint32_t above = 0;
        for (uint32_t i = 0; i < n; i++) above += e[i] > kth ? 1u : 0u;
        uint32_t ties = topK_ - above;
        for (uint32_t i = 0; i < n; i++) {
            if (e[i] > kth) continue;
            if (e[i] == kth && ties > 0) { ties--; continue; }
            e[i] = 0.f;
        }
        kept = topK_;
    }
    return kept;
}

void Sampler::beginCompletion() {
    std::fill(counts_.begin(), counts_.end(), 0u);
    completion_ = nextCompletionGeneration();
}

// Built without FMA (-O2, no -march): every step rounds to float32 as the device's __fadd_rn / __fmul_rn / __fsub_rn do.
void Sampler::applyControls(float *logits) const {
    const bool bias = !biasDense_.empty(), counted = !counts_.empty();
    for (uint32_t i = 0; i < vocabSize_; i++) {
        float x = logits[i];
        if (bias) x = x + biasDense_[i];
        if (counted && counts_[i] > 0) {
            const float pen = (float)counts_[i] * frequency_;
            x = x - pen;
            x = x - presence_;
        }
        logits[i] = x;
    }
}

int32_t Sampler::sample(float *logits) {
    if (!controlsActive()) return draw(logits);
    applyControls(logits);
    const int32_t token = draw(logits);
    counts_[token]++;
    return token;
}

int32_t Sampler::draw(float *logits) {
    const int n = (int)vocabSize_;
    if (temperature_ == 0.0f) {
        int best = 0;
        for (int i = 1; i < n; i++) if (logits[i] > logits[best]) best = i;
        return best;
    }
    // softmax with the shared exp (csrc/common/dl_expf.h) and an integer normaliser: bit-identical to the device sampler
    float mx = -INFINITY;
    for (int i = 0; i < n; i++) { logits[i] /= temperature_; mx = std::max(mx, logits[i]); }
    uint64_t sumFix = 0;
    for (int i = 0; i < n; i++) { logits[i] = expNeg(logits[i] - mx); sumFix += (uint64_t)(logits[i] * 1099511627776.0f); }
    int nS = n;   // |S|: the candidates left by the filters
    int single = -1;
    if (filtersActive()) {
        nS = (int)applyFilters(logits);
        sumFix = 0;
        for (int i = 0; i < n; i++) sumFix += (uint64_t)(logits[i] * 1099511627776.0f);
        if (nS == 1) {   // the one candidate: the lowest id holding the largest value
            single = 0;
            for (int i = 1; i < n; i++) if (logits[i] > logits[single]) single = i;
        }
    }
    const float inv = 1.0f / ((float)sumFix / 1099511627776.0f);
    for (int i = 0; i < n; i++) logits[i] *= inv;
    const float coin = rng_.nextF32();
    if (single >= 0) return single;
    // Prefix sums run in 2^-40 fixed point (64-bit integers): exact and order independent, so the device sampler
    // (csrc/cuda/sampler.cu), which adds the same terms in parallel, reaches the same decisions. The reference accumulates the same
    // sums in float (src/tokenizer.cpp:405-467); the two differ only when the coin falls within float rounding of a boundary.
    auto fix = [](float p) { return (uint64_t)(p * 1099511627776.0f); };
    if (topp_ <= 0.f || topp_ >= 1.f) {
        uint64_t cdf = 0;
        const uint64_t c = fix(coin);
        for (int i = 0; i < n; i++) { cdf += fix(logits[i]); if (c < cdf) return i; }
        return n - 1;
    }
    // nucleus: tokens below (1-p)/(n-1) can never be inside the top-p set, drop them before sorting
    const float cutoff = (1.0f - topp_) / (float)(nS - 1);
    candidates_.clear();
    for (int i = 0; i < n; i++) if (logits[i] >= cutoff) candidates_.push_back({logits[i], i});
    std::sort(candidates_.begin(), candidates_.end(), [](const std::pair<float, int32_t> &a, const std::pair<float, int32_t> &b) {
        return a.first > b.first || (a.first == b.first && a.second < b.second);
    });
    uint64_t cumulative = 0;
    const uint64_t target = fix(topp_);
    int last = (int)candidates_.size() - 1;
    for (int i = 0; i < (int)candidates_.size(); i++) {
        cumulative += fix(candidates_[i].first);
        if (cumulative > target) { last = i; break; }
    }
    const uint64_t r = fix(coin * ((float)cumulative / 1099511627776.0f));
    uint64_t cdf = 0;
    for (int i = 0; i <= last; i++) { cdf += fix(candidates_[i].first); if (r < cdf) return candidates_[i].second; }
    return candidates_[last].second;
}

// ---- chat templates --------------------------------------------------------------------------------

ChatTemplateType parseChatTemplateType(const std::string &name) {
    if (name == "llama2") return TEMPLATE_LLAMA2;
    if (name == "llama3") return TEMPLATE_LLAMA3;
    if (name == "deepSeek3") return TEMPLATE_DEEP_SEEK3;
    if (name == "chatml") return TEMPLATE_CHATML;
    throw std::runtime_error("Invalid chat template type: " + name);
}

const char *chatTemplateTypeName(ChatTemplateType t) {
    switch (t) {
        case TEMPLATE_LLAMA2: return "llama2";
        case TEMPLATE_LLAMA3: return "llama3";
        case TEMPLATE_DEEP_SEEK3: return "deepSeek3";
        case TEMPLATE_CHATML: return "chatml";
        default: return "unknown";
    }
}

ChatTemplateGenerator::ChatTemplateGenerator(ChatTemplateType type, const std::string &tpl, const std::string &eos)
    : type_(type), eos_(eos) {
    if (type_ == TEMPLATE_UNKNOWN) {
        if (tpl.empty()) throw std::runtime_error("The tokenizer does not include chat template");
        if (tpl.find("[INST]") != std::string::npos) type_ = TEMPLATE_LLAMA2;
        else if (tpl.find("<|start_header_id|>") != std::string::npos) type_ = TEMPLATE_LLAMA3;
        else if (tpl.find("<｜Assistant｜>") != std::string::npos) type_ = TEMPLATE_DEEP_SEEK3;
        else if (tpl.find("<|im_start|>") != std::string::npos) type_ = TEMPLATE_CHATML;
        else throw std::runtime_error("Not supported chat template");
    }
}

GeneratedChat ChatTemplateGenerator::generate(const std::vector<ChatItem> &items, bool gen) const {
    GeneratedChat out;
    std::string &b = out.content;
    const size_t n = items.size();
    if (type_ == TEMPLATE_LLAMA2) {
        size_t i = 0;
        if (n >= 2 && items[0].role == "system" && items[1].role == "user") {
            b += "[INST] <<SYS>>\n" + items[0].message + "\n<</SYS>>\n\n" + items[1].message + " [/INST]" + eos_;
            i = 2;
        }
        for (; i < n; i++) {
            if (items[i].role == "assistant") b += items[i].message + eos_;
            else if (items[i].role == "user") b += "[INST] " + items[i].message + " [/INST]" + eos_;
        }
    } else if (type_ == TEMPLATE_LLAMA3) {
        for (const ChatItem &it : items) b += "<|start_header_id|>" + it.role + "<|end_header_id|>\n\n" + it.message + eos_;
        if (gen) b += "<|start_header_id|>assistant<|end_header_id|>\n\n";
    } else if (type_ == TEMPLATE_DEEP_SEEK3) {
        size_t i = 0;
        if (n > 0 && items[0].role == "system") { b += items[0].message; i = 1; }
        for (; i < n; i++) {
            if (items[i].role == "user") b += "<｜User｜>" + items[i].message;
            else if (items[i].role == "assistant") b += "<｜Assistant｜>" + items[i].message;
        }
        if (gen) {
            b += "<｜Assistant｜><think>\n";
            out.publicPrompt = "<think>\n";
        }
    } else if (type_ == TEMPLATE_CHATML) {
        for (const ChatItem &it : items)
            if (it.role == "system" || it.role == "user" || it.role == "assistant")
                b += "<|im_start|>" + it.role + "\n" + it.message + "<|im_end|>\n";
        if (gen) b += "<|im_start|>assistant\n";
    }
    return out;
}

// ---- stop detector -----------------------------------------------------------------------------------

EosDetector::EosDetector(std::vector<int32_t> tokens, std::vector<std::string> pieces, int padLeft, int padRight)
    : tokens_(std::move(tokens)), pieces_(std::move(pieces)), padLeft_(padLeft), padRight_(padRight) {
    if (tokens_.size() != pieces_.size()) throw std::invalid_argument("EosDetector: tokens/pieces size mismatch");
}

bool EosDetector::isEos(int32_t tokenId) const {
    return std::find(tokens_.begin(), tokens_.end(), tokenId) != tokens_.end();
}

EosDetectorResult EosDetector::append(int32_t tokenId, const std::string &piece) {
    buffer_ += piece;
    if (isEos(tokenId)) {
        eosPos_ = (int)buffer_.size();
        return EOS;
    }
    eosPos_ = -1;
    const long len = (long)buffer_.size();
    for (const std::string &stop : pieces_) {
        const long ps = (long)stop.size();
        if (len > ps + padLeft_ + padRight_) continue;
        for (long lo = 0; lo <= padLeft_; lo++) {
            long n = len - lo;
            if (n <= 0 || n > ps + padRight_) continue;
            if (n > ps) n = ps;
            if (buffer_.compare(lo, n, stop, 0, n) == 0) {
                if (n == ps) {
                    eosPos_ = (int)lo;
                    buffer_.resize(lo);
                    return EOS;
                }
                return MAYBE_EOS;
            }
        }
    }
    return NOT_EOS;
}

std::string EosDetector::getDelta() const {
    if (buffer_.empty() || eosPos_ == 0) return std::string();
    return buffer_;
}

void EosDetector::reset() { buffer_.clear(); }

// ---- stop strings ---------------------------------------------------------------------------------------------------

StopMatcher::StopMatcher(std::vector<std::string> stops) : stops_(std::move(stops)) {
    for (const std::string &s : stops_)
        if (s.empty()) throw std::invalid_argument("StopMatcher: empty stop string");
}

// No occurrence existed before this delta, and every occurrence that ends inside it starts inside the held bytes or the delta
// (the held bytes are the longest suffix of G that is a proper prefix of a stop string), so searching held + delta is enough.
std::string StopMatcher::push(const std::string &delta) {
    if (stopped_) return std::string();
    std::string text;
    text.reserve(held_.size() + delta.size());
    text += held_;
    text += delta;
    held_.clear();
    size_t cut = std::string::npos;
    for (const std::string &s : stops_) cut = std::min(cut, text.find(s));
    if (cut != std::string::npos) {
        stopped_ = true;
        text.resize(cut);
        return text;
    }
    size_t hold = 0;
    for (const std::string &s : stops_) {
        for (size_t l = std::min(text.size(), s.size() - 1); l > hold; l--)
            if (text[text.size() - l] == s[0] && text.compare(text.size() - l, l, s, 0, l) == 0) { hold = l; break; }
    }
    held_.assign(text, text.size() - hold, hold);
    text.resize(text.size() - hold);
    return text;
}

std::string StopMatcher::flush() {
    std::string out;
    out.swap(held_);
    return out;
}

}  // namespace dl
