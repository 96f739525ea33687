#include "api_server.hpp"
#include "../host/slot_scheduler.hpp"

#include <arpa/inet.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/socket.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <optional>
#include <stdexcept>

namespace dl {

// ---- HTTP plumbing ----------------------------------------------------------------------------------------------------

void HttpRequest::send(const std::string &data) const {
    size_t off = 0;
    while (off < data.size()) {
        const ssize_t n = ::send(fd, data.data() + off, data.size() - off, MSG_NOSIGNAL);
        if (n <= 0) throw std::runtime_error("Error while writing to socket");
        off += (size_t)n;
    }
}

HttpRequest HttpRequest::read(int fd) {
    HttpRequest req;
    req.fd = fd;
    std::string data;
    char buf[8192];
    size_t headEnd = std::string::npos, sepLen = 0;
    while (true) {
        const size_t a = data.find("\r\n\r\n"), b = data.find("\n\n");
        if (a != std::string::npos && (b == std::string::npos || a <= b)) { headEnd = a; sepLen = 4; break; }
        if (b != std::string::npos) { headEnd = b; sepLen = 2; break; }
        const ssize_t n = ::recv(fd, buf, sizeof(buf), 0);
        if (n <= 0) throw std::runtime_error("Error while reading headers from socket");
        data.append(buf, (size_t)n);
        if (data.size() > (1u << 20)) throw std::runtime_error("Request header too large");
    }
    const std::string head = data.substr(0, headEnd);
    std::string rest = data.substr(headEnd + sepLen);
    size_t lineStart = 0;
    bool first = true;
    while (lineStart <= head.size()) {
        size_t lineEnd = head.find('\n', lineStart);
        if (lineEnd == std::string::npos) lineEnd = head.size();
        std::string line = head.substr(lineStart, lineEnd - lineStart);
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (first) {
            const size_t s1 = line.find(' ');
            if (s1 != std::string::npos) {
                size_t s2 = line.find(' ', s1 + 1);
                if (s2 == std::string::npos) s2 = line.size();
                req.method = line.substr(0, s1);
                for (char &c : req.method) c = (char)std::toupper((unsigned char)c);
                req.path = line.substr(s1 + 1, s2 - s1 - 1);
            }
            first = false;
        } else {
            const size_t colon = line.find(':');
            if (colon != std::string::npos) {
                std::string k = line.substr(0, colon), v = line.substr(colon + 1);
                for (char &c : k) c = (char)std::tolower((unsigned char)c);
                const auto trim = [](std::string &s) {
                    while (!s.empty() && std::isspace((unsigned char)s.back())) s.pop_back();
                    size_t i = 0;
                    while (i < s.size() && std::isspace((unsigned char)s[i])) i++;
                    s.erase(0, i);
                };
                trim(k); trim(v);
                req.headers[k] = v;
            }
        }
        lineStart = lineEnd + 1;
    }
    size_t length = 0;
    const auto it = req.headers.find("content-length");
    if (it != req.headers.end() && !it->second.empty()) length = (size_t)std::strtoull(it->second.c_str(), nullptr, 10);
    if (length > (64u << 20)) throw std::runtime_error("Request body too large");
    if (length > 0 && rest.size() > length) throw std::runtime_error("Received more body data than Content-Length header said");
    while (rest.size() < length) {
        const ssize_t n = ::recv(fd, buf, std::min(sizeof(buf), length - rest.size()), 0);
        if (n <= 0) throw std::runtime_error("Error while reading body from socket");
        rest.append(buf, (size_t)n);
    }
    req.body = rest;
    if (!rest.empty()) {
        req.json = JsonParser(req.body).parse();
        req.hasJson = true;
    }
    return req;
}

void HttpRequest::writeCors() const {
    send("HTTP/1.1 204 No Content\r\nAccess-Control-Allow-Origin: *\r\nAccess-Control-Allow-Methods: GET, POST, PUT, DELETE\r\n"
         "Access-Control-Allow-Headers: Content-Type, Authorization\r\nConnection: close\r\n\r\n");
}
void HttpRequest::writeNotFound() const { send("HTTP/1.1 404 Not Found\r\nConnection: close\r\nContent-Length: 9\r\n\r\nNot Found"); }
void HttpRequest::writeJson(const std::string &text) const {
    send("HTTP/1.1 200 OK\r\nAccess-Control-Allow-Origin: *\r\nContent-Type: application/json; charset=utf-8\r\nConnection: close\r\n"
         "Content-Length: " + std::to_string(text.size()) + "\r\n\r\n" + text);
}
void HttpRequest::writeStreamStart() const {
    send("HTTP/1.1 200 OK\r\nAccess-Control-Allow-Origin: *\r\nContent-Type: text/event-stream; charset=utf-8\r\nConnection: close\r\n"
         "Transfer-Encoding: chunked\r\n\r\n");
}
void HttpRequest::writeStreamChunk(const std::string &data) const {
    char len[32];
    std::snprintf(len, sizeof(len), "%zx\r\n", data.size());
    send(std::string(len) + data + "\r\n");
}
void HttpRequest::writeStreamEnd() const { send("0000\r\n\r\n"); }

// ---- NaiveCache ---------------------------------------------------------------------------------------------------------

uint32_t NaiveCache::resolveDeltaPrompt(std::vector<ChatItem> &messages) {
    const size_t n = items_.size();
    if (n == 0) return 0;
    if (messages.size() > n) {
        bool prefix = true;
        for (size_t i = 0; i < n && prefix; i++)
            prefix = items_[i].msg.role == messages[i].role && items_[i].msg.message == messages[i].message;
        if (prefix) {
            const uint32_t start = items_[n - 1].endPos;
            std::printf("🐤 Found naive cache for %zu messages, pos=%u\n", n, start);
            messages.erase(messages.begin(), messages.begin() + (long)n);
            return start;
        }
    }
    clear();
    return 0;
}

size_t NaiveCache::coveredPrefix(const std::vector<ChatItem> &messages) const {
    const size_t n = items_.size();
    if (messages.size() <= n) return 0;
    for (size_t i = 0; i < n; i++)
        if (items_[i].msg.role != messages[i].role || items_[i].msg.message != messages[i].message) return 0;
    return n;
}

namespace {
std::string joinEntries(const std::vector<std::string> &entries) {
    std::string s = "{\"content\": [";
    for (size_t i = 0; i < entries.size(); i++) s += (i ? ", " : "") + entries[i];
    return s + "]}";
}
}  // namespace

std::string chunkJson(const std::string *delta, bool stop, uint32_t index, const std::vector<std::string> *logprobs) {
    std::string s = "{\"id\": \"cmpl-c0\", \"object\": \"chat.completion\", \"created\": " + std::to_string((long long)std::time(nullptr)) +
                    ", \"model\": \"Distributed Model\", \"choices\": [{\"index\": " + std::to_string(index) + ", \"finish_reason\": " +
                    (stop ? "\"stop\"" : "\"\"");
    if (!stop) s += ", \"delta\": {\"role\": \"assistant\", \"content\": " + jsonEscape(delta ? *delta : std::string()) + "}";
    if (!stop && logprobs) s += ", \"logprobs\": " + joinEntries(*logprobs);
    s += "}]}";
    return s;
}

// ---- log-probabilities --------------------------------------------------------------------------------------------------------

TokenLogprobs decodeLogprobs(const int32_t *w) {
    const auto f = [](int32_t bits) { float v; std::memcpy(&v, &bits, 4); return v; };
    TokenLogprobs e;
    e.token = w[0];
    e.logprob = f(w[1]);
    for (int j = 0; j < w[2]; j++) e.top.push_back({w[4 + 2 * j], f(w[5 + 2 * j])});
    return e;
}

namespace {
// Strict UTF-8 (no overlong forms, surrogates or code points above U+10FFFF): what Python accepts when it decodes a request body.
bool validUtf8(const std::string &s) {
    for (size_t i = 0; i < s.size();) {
        const unsigned char c = (unsigned char)s[i];
        int need;
        unsigned char lo = 0x80, hi = 0xbf;
        if (c < 0x80) { i++; continue; }
        else if (c >= 0xc2 && c <= 0xdf) need = 1;
        else if (c >= 0xe0 && c <= 0xef) { need = 2; if (c == 0xe0) lo = 0xa0; else if (c == 0xed) hi = 0x9f; }
        else if (c >= 0xf0 && c <= 0xf4) { need = 3; if (c == 0xf0) lo = 0x90; else if (c == 0xf4) hi = 0x8f; }
        else return false;
        if (i + (size_t)need >= s.size()) return false;
        for (int k = 1; k <= need; k++) {
            const unsigned char d = (unsigned char)s[i + (size_t)k];
            if (d < (k == 1 ? lo : 0x80) || d > (k == 1 ? hi : 0xbf)) return false;
        }
        i += (size_t)need + 1;
    }
    return true;
}
}  // namespace

std::vector<std::string> parseStop(const JsonValue &body) {
    const JsonValue *v = body.find("stop");
    std::vector<std::string> out;
    if (!v || v->kind == JsonValue::Null) return out;
    const auto take = [&](const JsonValue &s) {
        if (s.kind != JsonValue::String || s.loneSurrogate || s.str.empty() || s.str.size() > kMaxStopBytes || !validUtf8(s.str))
            throw std::runtime_error("'stop' strings must be 1 to 256 bytes of UTF-8");
        out.push_back(s.str);
    };
    if (v->kind == JsonValue::String) take(*v);
    else if (v->kind == JsonValue::Array && v->arr.size() <= kMaxStopStrings) for (const JsonValue &s : v->arr) take(s);
    else throw std::runtime_error("'stop' must be a string or an array of at most 4 strings");
    return out;
}

int parseLogprobs(const JsonValue &body) {
    const JsonValue *on = body.find("logprobs"), *k = body.find("top_logprobs");
    if (on && on->kind != JsonValue::Bool) throw std::runtime_error("'logprobs' must be a boolean");
    const bool enabled = on && on->b;
    if (k && !enabled) throw std::runtime_error("'top_logprobs' needs 'logprobs': true");
    if (k && !(k->kind == JsonValue::Number && k->integral && k->num >= 0 && k->num <= kMaxTopLogprobs))
        throw std::runtime_error("'top_logprobs' must be an integer from 0 to 20");
    return enabled ? (k ? (int)k->num : 0) : -1;
}

namespace {
// repr() of a Python float: the shortest digits that read back as v, positional for exponents -4 .. 15, else d.ddde±XX
std::string pyFloat(double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v < 0 ? "-Infinity" : "Infinity";
    if (v == 0) return std::signbit(v) ? "-0.0" : "0.0";
    char buf[64];
    for (int p = 1; p <= 17; p++) {
        std::snprintf(buf, sizeof(buf), "%.*e", p - 1, v);
        if (std::strtod(buf, nullptr) == v) break;
    }
    std::string s(buf), sign;
    if (s[0] == '-') { sign = "-"; s = s.substr(1); }
    const size_t ePos = s.find('e');
    const int e = std::atoi(s.c_str() + ePos + 1);
    std::string digits;
    for (size_t i = 0; i < ePos; i++) if (s[i] != '.') digits += s[i];
    while (digits.size() > 1 && digits.back() == '0') digits.pop_back();
    if (e >= -4 && e < 16) {
        if (e < 0) return sign + "0." + std::string((size_t)(-e - 1), '0') + digits;
        if (digits.size() <= (size_t)e + 1) return sign + digits + std::string((size_t)e + 1 - digits.size(), '0') + ".0";
        return sign + digits.substr(0, (size_t)e + 1) + "." + digits.substr((size_t)e + 1);
    }
    std::snprintf(buf, sizeof(buf), "e%c%02d", e < 0 ? '-' : '+', std::abs(e));
    return sign + digits.substr(0, 1) + (digits.size() > 1 ? "." + digits.substr(1) : "") + buf;
}

// bytes decoded as UTF-8 with replacement (one U+FFFD per maximal invalid subpart, as Python's errors="replace"), then escaped as
// json.dumps does by default: every character outside ' '..'~' as \uXXXX (surrogate pairs above U+FFFF)
std::string jsonEscapeUtf8Ascii(const std::string &bytes) {
    std::string out = "\"";
    const auto put = [&](uint32_t cp) {
        char buf[16];
        if (cp == '"') out += "\\\"";
        else if (cp == '\\') out += "\\\\";
        else if (cp == '\n') out += "\\n";
        else if (cp == '\r') out += "\\r";
        else if (cp == '\t') out += "\\t";
        else if (cp == '\b') out += "\\b";
        else if (cp == '\f') out += "\\f";
        else if (cp >= 0x20 && cp < 0x7f) out += (char)cp;
        else if (cp < 0x10000) { std::snprintf(buf, sizeof(buf), "\\u%04x", cp); out += buf; }
        else {
            const uint32_t c = cp - 0x10000;
            std::snprintf(buf, sizeof(buf), "\\u%04x\\u%04x", 0xd800 + (c >> 10), 0xdc00 + (c & 0x3ff));
            out += buf;
        }
    };
    const size_t n = bytes.size();
    for (size_t i = 0; i < n;) {
        const unsigned char c = (unsigned char)bytes[i];
        int need;
        uint32_t cp;
        if (c < 0x80) { put(c); i++; continue; }
        else if (c >= 0xc2 && c <= 0xdf) { need = 1; cp = c & 0x1f; }
        else if (c >= 0xe0 && c <= 0xef) { need = 2; cp = c & 0x0f; }
        else if (c >= 0xf0 && c <= 0xf4) { need = 3; cp = c & 0x07; }
        else { put(0xfffd); i++; continue; }
        size_t j = i + 1;
        int got = 0;
        for (; got < need && j < n; got++, j++) {
            const unsigned char d = (unsigned char)bytes[j];
            unsigned char lo = 0x80, hi = 0xbf;
            if (got == 0) {
                if (c == 0xe0) lo = 0xa0;
                else if (c == 0xed) hi = 0x9f;
                else if (c == 0xf0) lo = 0x90;
                else if (c == 0xf4) hi = 0x8f;
            }
            if (d < lo || d > hi) break;
            cp = (cp << 6) | (d & 0x3f);
        }
        if (got == need) put(cp);
        else put(0xfffd);
        i = j;
    }
    return out + "\"";
}

std::string tokenJson(const Tokenizer &tok, int32_t id, float logprob) {
    const std::string &b = tok.data().vocab.at((size_t)id);
    std::string bytes;
    for (size_t i = 0; i < b.size(); i++) bytes += (i ? ", " : "") + std::to_string((unsigned)(unsigned char)b[i]);
    return "{\"token\": " + jsonEscapeUtf8Ascii(b) + ", \"logprob\": " + pyFloat((double)logprob) + ", \"bytes\": [" + bytes + "]";
}
}  // namespace

std::string logprobEntryJson(const Tokenizer &tok, const TokenLogprobs &e) {
    std::string s = tokenJson(tok, e.token, e.logprob) + ", \"top_logprobs\": [";
    for (size_t i = 0; i < e.top.size(); i++) s += (i ? ", " : "") + tokenJson(tok, e.top[i].first, e.top[i].second) + "}";
    return s + "]}";
}

namespace {
// Entries of the tokens of n choices: all of them for the final JSON, those not yet sent for the stream. The token that ends a
// choice by end of sequence gets none (the Python server's LogprobsLog).
struct LogprobsLog {
    std::vector<std::string> next;
    std::vector<std::vector<std::string>> all, pending;
    explicit LogprobsLog(uint32_t n = 0) : next(n), all(n), pending(n) {}
    void consumed(uint32_t i, bool eos) {
        if (!eos) { all[i].push_back(next[i]); pending[i].push_back(next[i]); }
        next[i].clear();
    }
    std::vector<std::string> take(uint32_t i) { std::vector<std::string> out; out.swap(pending[i]); return out; }
};

// choice i's stop chunk, after one delta chunk with empty content for entries still unsent
void writeStreamFinish(const HttpRequest &req, uint32_t i, LogprobsLog *lps) {
    if (lps && !lps->pending[i].empty()) {
        const std::string empty;
        const std::vector<std::string> e = lps->take(i);
        req.writeStreamChunk("data: " + chunkJson(&empty, false, i, &e) + "\r\n\r\n");
    }
    req.writeStreamChunk("data: " + chunkJson(nullptr, true, i) + "\r\n\r\n");
}

std::string choiceJson(uint32_t i, const std::string &content, const LogprobsLog *lps) {
    return "{\"index\": " + std::to_string(i) + ", \"message\": {\"role\": \"assistant\", \"content\": " + jsonEscape(content) +
           "}, \"finish_reason\": \"stop\"" + (lps ? ", \"logprobs\": " + joinEntries(lps->all[i]) : std::string()) + "}";
}
}  // namespace

// ---- several completions of one prompt ------------------------------------------------------------------------------------

std::vector<std::vector<int32_t>> runChoices(InferenceBackend &backend, int32_t token, uint32_t P, uint32_t n, int maxTokens, uint32_t seqLen,
                                             Sampler &sampler, uint64_t baseSeed, const std::function<bool(uint32_t, int32_t)> &onToken,
                                             const std::function<void(uint32_t, const TokenLogprobs &)> &onLogprobs) {
    if (n < 1 || n > kMaxChoices) throw std::runtime_error("n must be between 1 and 8");
    std::vector<std::vector<int32_t>> out(n);
    const uint32_t C = P + 1 < seqLen ? (seqLen - 1 - P) / n : 0;
    uint32_t limit = n == 1 ? (P < seqLen ? seqLen - P : 0) : C;
    if (maxTokens > 0) limit = std::min<uint32_t>((uint32_t)maxTokens, limit);
    if (limit == 0) return out;
    sampler.beginCompletion();
    // today's single-sequence path from P for the choices in [first, last]; they all see the same tokens
    const auto single = [&](Sampler &smp, uint32_t first, uint32_t last) {
        int32_t tok = token;
        uint32_t pos = P;
        std::vector<bool> done(n, false);
        uint32_t nDone = 0;
        // a single greedy completion with a draft model takes speculative rounds of several tokens (the same tokens)
        const bool spec = n == 1 && !onLogprobs && backend.speculates(smp);
        while (out[first].size() < limit) {
            const std::vector<int32_t> toks = spec ? backend.specRound(tok, pos) : std::vector<int32_t>{backend.next(tok, pos, smp)};
            const TokenLogprobs entry = onLogprobs ? backend.lastLogprobs().at(0) : TokenLogprobs();
            for (const int32_t t : toks) {
                tok = t;
                pos++;
                for (uint32_t i = first; i <= last; i++) {
                    if (done[i]) continue;
                    out[i].push_back(tok);
                    if (onLogprobs) onLogprobs(i, entry);
                    if (onToken(i, tok)) { done[i] = true; nDone++; }
                }
                if (nDone == last - first + 1 || out[first].size() >= limit) break;
            }
            if (nDone == last - first + 1) break;
        }
    };
    if (n == 1 || sampler.temperature() == 0.f) {   // greedy choices are all equal: one run
        single(sampler, 0, n - 1);
        return out;
    }
    const float T = sampler.temperature(), topp = sampler.topp();
    std::vector<uint64_t> seeds(n);
    for (uint32_t i = 0; i < n; i++) seeds[i] = choiceSeed(baseSeed, i);
    if (!backend.batchedChoices(n)) {
        const uint64_t saved = backend.saveSampler();
        for (uint32_t i = 0; i < n; i++) {
            Sampler smp(sampler.vocabSize(), T, topp, seeds[i]);   // a fresh sampler: its own counts, from zero
            smp.setControls(sampler.presencePenalty(), sampler.frequencyPenalty(), sampler.logitBias());
            smp.setFilters(sampler.topK(), sampler.minP());
            single(smp, i, i);
        }
        backend.restoreSampler(saved);
        return out;
    }
    backend.seedChoices(seeds);
    backend.choiceControls(sampler, n);
    std::vector<int32_t> last = backend.choicesFirst(token, P, n, T, topp);
    uint32_t active = (1u << n) - 1u;
    for (uint32_t j = 0;; j++) {
        const std::vector<TokenLogprobs> entries = onLogprobs ? backend.lastLogprobs() : std::vector<TokenLogprobs>();
        for (uint32_t i = 0; i < n; i++) {
            if (!((active >> i) & 1u)) continue;
            out[i].push_back(last[i]);
            if (onLogprobs) onLogprobs(i, entries.at(i));
            if (onToken(i, last[i]) || out[i].size() >= limit) active &= ~(1u << i);
        }
        if (!active) break;
        last = backend.choicesStep(last, P, C, j, active, T, topp);
    }
    return out;
}

// ---- completion -----------------------------------------------------------------------------------------------------------

namespace {
std::vector<std::string> stopPieces(const Tokenizer &tok) {
    std::vector<std::string> out;
    for (int32_t id : tok.data().eosIds) out.push_back(tok.data().vocab[(size_t)id]);
    return out;
}
int maxLen(const std::vector<std::string> &v) {
    size_t m = 0;
    for (const std::string &s : v) m = std::max(m, s.size());
    return (int)m;
}
float boundedNumber(const JsonValue &v, double limit, const char *what) {
    if (v.kind != JsonValue::Number || !(v.num >= -limit && v.num <= limit))
        throw std::runtime_error(std::string("'") + what + "' must be a number from " + std::to_string((int)-limit) + " to " + std::to_string((int)limit));
    return (float)v.num;
}
// The request's sampling controls; same rules as distributed_llama_b200.apps.api_server.parse_controls: penalties are numbers in
// [-2, 2] (absent: the server's defaults); logit_bias is an object of at most 100 entries whose keys are decimal token ids in
// [0, vocab) without leading zeros and whose values are numbers in [-100, 100]. A repeated key keeps its last value.
void parseControls(const JsonValue &body, uint32_t vocab, float &presence, float &frequency, std::vector<std::pair<int32_t, float>> &bias) {
    if (const JsonValue *v = body.find("presence_penalty")) presence = boundedNumber(*v, kMaxPenalty, "presence_penalty");
    if (const JsonValue *v = body.find("frequency_penalty")) frequency = boundedNumber(*v, kMaxPenalty, "frequency_penalty");
    bias.clear();
    const JsonValue *b = body.find("logit_bias");
    if (!b) return;
    if (!b->isObject()) throw std::runtime_error("'logit_bias' must be an object");
    std::map<int32_t, float> byId;
    for (const auto &kv : b->obj) {
        const std::string &k = kv.first;
        bool ok = !k.empty() && k.size() <= 10 && (k[0] != '0' || k.size() == 1);
        for (char c : k) ok = ok && c >= '0' && c <= '9';
        if (!ok || std::stoull(k) >= vocab) throw std::runtime_error("'logit_bias' keys must be token ids below the vocabulary size");
        byId[(int32_t)std::stoull(k)] = boundedNumber(kv.second, kMaxLogitBias, "logit_bias");
    }
    if (byId.size() > kMaxLogitBiasEntries) throw std::runtime_error("'logit_bias' has more than 100 entries");
    bias.assign(byId.begin(), byId.end());
}

}  // namespace

void parseFilters(const JsonValue &body, uint32_t &topK, float &minP) {
    if (const JsonValue *v = body.find("top_k")) {
        if (!(v->kind == JsonValue::Number && v->integral && v->num >= 0 && v->num <= (double)kMaxTopK))
            throw std::runtime_error("'top_k' must be an integer from 0 to 2147483647");
        topK = (uint32_t)v->num;
    }
    if (const JsonValue *v = body.find("min_p")) {
        if (!(v->kind == JsonValue::Number && v->num >= 0 && v->num <= 1)) throw std::runtime_error("'min_p' must be a number from 0 to 1");
        minP = (float)v->num;
    }
}

namespace {

// A validated chat completion request: the rules of distributed_llama_b200.apps.api_server.parse_chat, except that a number field
// that is not a number counts as absent.
struct ChatRequest {
    std::vector<ChatItem> messages;
    bool stream = false, hasSeed = false;
    uint32_t n = 1;
    int maxTokens = -1;
    int logprobs = -1;   // top_logprobs k, -1: none
    float temperature = 0.f, topp = 0.9f, presence = 0.f, frequency = 0.f;
    std::vector<std::pair<int32_t, float>> bias;
    uint32_t topK = 0;   // sampling filters (parseFilters)
    float minP = 0.f;
    uint64_t seed = 0;
    std::vector<std::string> stop;   // parseStop
};

// maxN: the largest `n` (the slot count under --parallel)
ChatRequest parseChat(const JsonValue &body, const ApiConfig &cfg, uint32_t vocab, uint32_t maxN) {
    if (!body.isObject()) throw std::runtime_error("request body must be a JSON object");
    ChatRequest c;
    if (const JsonValue *v = body.find("n")) {
        if (v->kind != JsonValue::Number || v->num != (double)(int64_t)v->num || v->num < 1 || v->num > kMaxChoices)
            throw std::runtime_error("'n' must be an integer from 1 to 8");
        c.n = (uint32_t)v->num;
    }
    if (c.n > maxN) throw std::runtime_error("'n' must not exceed --parallel");
    c.presence = cfg.presencePenalty;
    c.frequency = cfg.frequencyPenalty;
    parseControls(body, vocab, c.presence, c.frequency, c.bias);
    c.topK = cfg.topK;
    c.minP = cfg.minP;
    parseFilters(body, c.topK, c.minP);
    c.logprobs = parseLogprobs(body);
    c.stop = parseStop(body);
    for (const JsonValue &m : body.at("messages").arr) c.messages.push_back({m.at("role").str, m.at("content").str});
    c.stream = body.boolOr("stream", false);
    c.temperature = (float)body.numberOr("temperature", cfg.temperature);
    if (c.temperature < 0.f) throw std::runtime_error("'temperature' must not be negative");
    c.topp = (float)body.numberOr("top_p", cfg.topp);
    if (const JsonValue *sd = body.find("seed")) if (sd->kind == JsonValue::Number) { c.seed = (uint64_t)sd->num; c.hasSeed = true; }
    c.maxTokens = (int)body.numberOr("max_tokens", -1);
    return c;
}

std::string completionJson(uint32_t nPrompt, const std::vector<std::vector<int32_t>> &out, const std::vector<std::string> &buffers,
                           const LogprobsLog *lps) {
    uint32_t nCompletion = 0;
    std::string choices;
    for (uint32_t i = 0; i < buffers.size(); i++) {
        nCompletion += (uint32_t)out[i].size();
        choices += std::string(i ? ", " : "") + choiceJson(i, buffers[i], lps);
    }
    return "{\"id\": \"cmpl-j0\", \"object\": \"chat.completion\", \"created\": " + std::to_string((long long)std::time(nullptr)) +
           ", \"model\": \"Distributed Model\", \"usage\": {\"completion_tokens\": " + std::to_string(nCompletion) +
           ", \"prompt_tokens\": " + std::to_string(nPrompt) + ", \"total_tokens\": " + std::to_string(nPrompt + nCompletion) +
           "}, \"choices\": [" + choices + "]}";
}

// The response to one chat request: its n choices' decoders, stop detectors, texts and log-probability entries, written as stream
// chunks or as one cmpl-j0 JSON body (the Python server's ChatResponse). With `stop` strings each choice also has a StopMatcher
// after its detector. echo: print the tokens' pieces to stdout.
class ChatResponse {
public:
    ChatResponse(const HttpRequest &req, const ChatRequest &chat, const Tokenizer &tok, const std::vector<std::string> &stops, bool echo = false)
        : req_(req), tok_(tok), n_(chat.n), stream_(chat.stream), echo_(echo), hasLog_(chat.logprobs >= 0), log_(chat.n),
          dets_(chat.n, EosDetector(tok.data().eosIds, stops, maxLen(stops), maxLen(stops))), pending_(chat.n), buffers_(chat.n) {
        if (!chat.stop.empty()) matchers_.assign(chat.n, StopMatcher(chat.stop));
    }
    // choice i's content so far, bytes held back by its matcher included
    std::string text(uint32_t i) const { return matchers_.empty() ? buffers_[i] : buffers_[i] + matchers_[i].held(); }
    // choice i ended at a stop string
    bool stopped(uint32_t i) const { return !matchers_.empty() && matchers_[i].stopped(); }
    // every choice's text starts with the prompt's public part; a stream sends its head and that part
    void start(const std::string &publicPrompt) {
        buffers_.assign(n_, publicPrompt);
        if (!stream_) return;
        req_.writeStreamStart();
        if (!publicPrompt.empty())
            for (uint32_t i = 0; i < n_; i++) chunk(i, publicPrompt);
    }
    void onLogprobs(uint32_t i, const TokenLogprobs &e) { log_.next[i] = logprobEntryJson(tok_, e); }
    // choice i's next token; true when it ended the choice (end of sequence or stop string)
    bool onToken(uint32_t i, int32_t t) {
        const std::string piece = tok_.decodeWith(pending_[i], t);
        if (echo_ && !piece.empty()) { std::printf("%s", piece.c_str()); std::fflush(stdout); }
        const EosDetectorResult kind = dets_[i].append(t, piece);
        if (hasLog_) log_.consumed(i, kind == EOS);
        if (kind == NOT_EOS || kind == EOS) {
            std::string delta = dets_[i].getDelta();
            if (!matchers_.empty()) delta = matchers_[i].push(delta);
            if (!delta.empty()) {
                if (stream_) chunk(i, delta);
                buffers_[i] += delta;
            }
            dets_[i].reset();
        }
        return kind == EOS || stopped(i);
    }
    // every choice is done (out[i]: choice i's tokens): the stop chunks and [DONE], or the JSON body. Bytes a matcher still holds
    // (a choice that ended another way) join the text, in one delta chunk before the stop chunk of a stream.
    void finish(const std::vector<std::vector<int32_t>> &out, uint32_t nPrompt) {
        for (uint32_t i = 0; i < n_; i++) {
            const std::string rest = matchers_.empty() ? std::string() : matchers_[i].flush();
            buffers_[i] += rest;
            if (!stream_) continue;
            if (!rest.empty()) chunk(i, rest);
            writeStreamFinish(req_, i, lps());
        }
        if (!stream_) { req_.writeJson(completionJson(nPrompt, out, buffers_, lps())); return; }
        req_.writeStreamChunk("data: [DONE]");
        req_.writeStreamEnd();
    }
private:
    LogprobsLog *lps() { return hasLog_ ? &log_ : nullptr; }
    void chunk(uint32_t i, const std::string &text) {
        const std::vector<std::string> e = hasLog_ ? log_.take(i) : std::vector<std::string>();
        req_.writeStreamChunk("data: " + chunkJson(&text, false, i, hasLog_ ? &e : nullptr) + "\r\n\r\n");
    }
    const HttpRequest &req_;
    const Tokenizer &tok_;
    uint32_t n_;
    bool stream_, echo_, hasLog_;
    LogprobsLog log_;
    std::vector<EosDetector> dets_;
    std::vector<StopMatcher> matchers_;   // empty without `stop`
    std::vector<std::string> pending_, buffers_;
};

// A prompt resolved against a NaiveCache (the tokens to prefill from `start`, the last prompt token at P), the prompt's token count
// and its public part.
struct Prompt : SlotPrompt {
    uint32_t nPrompt = 0;
    std::string publicPrompt;
};

// Resolves `messages` against `cache` and records the messages still to be evaluated in it. echo: print the prompt to stdout.
Prompt preparePrompt(const ChatTemplateGenerator &gen, const Tokenizer &tok, NaiveCache &cache, std::vector<ChatItem> messages, uint32_t ctxLen,
                     bool echo = false) {
    Prompt p;
    p.start = cache.resolveDeltaPrompt(messages);
    const GeneratedChat g = gen.generate(messages, true);
    if (echo) std::printf("🔹%s🔸", g.content.c_str());
    const std::vector<int32_t> tokens = tok.encode(g.content, p.start == 0, true);
    p.nPrompt = (uint32_t)tokens.size();
    p.P = std::min(p.start + p.nPrompt - 1, ctxLen);
    for (const ChatItem &m : messages) cache.push(p.P, m);
    const uint32_t nPref = p.P - p.start;
    p.prefill.assign(tokens.begin(), tokens.begin() + nPref);
    p.token = nPref < tokens.size() ? tokens[nPref] : tokens.back();
    p.publicPrompt = g.publicPrompt;
    return p;
}

// After a single completion of the prompt ending at P the cache keeps its answer too, unless it filled the context.
void rememberAnswer(NaiveCache &cache, uint32_t P, size_t nOut, const std::string &text, uint32_t ctxLen) {
    const uint32_t end = P + (uint32_t)nOut;
    if (end == ctxLen) cache.clear();
    else cache.push(end, {"assistant", text});
}
}  // namespace

float parsePenalty(const std::string &flag, const std::string &value) {
    const float v = std::stof(value);
    if (!(v >= -kMaxPenalty && v <= kMaxPenalty)) throw std::runtime_error(flag + " must be from -2 to 2");
    return v;
}

uint32_t parseTopK(const std::string &flag, const std::string &value) {
    bool ok = !value.empty() && value.size() <= 10;
    for (char c : value) ok = ok && c >= '0' && c <= '9';
    if (!ok || std::stoull(value) > kMaxTopK) throw std::runtime_error(flag + " must be an integer from 0 to 2147483647");
    return (uint32_t)std::stoull(value);
}

float parseMinP(const std::string &flag, const std::string &value) {
    const float v = std::stof(value);
    if (!(v >= 0.f && v <= 1.f)) throw std::runtime_error(flag + " must be from 0 to 1");
    return v;
}

ApiServer::ApiServer(InferenceBackend &backend, Tokenizer &tokenizer, const ApiConfig &cfg)
    : backend_(backend), tok_(tokenizer), cfg_(cfg), sampler_(std::min<uint32_t>(backend.vocabSize(), tokenizer.vocabSize()), cfg.temperature, cfg.topp, cfg.seed),
      stops_(stopPieces(tokenizer)),
      gen_(cfg.chatTemplate.empty() ? TEMPLATE_UNKNOWN : parseChatTemplateType(cfg.chatTemplate), tokenizer.data().chatTemplate,
           stops_.empty() ? std::string() : stops_[0]) {
    backend_.setVocabLimit(tokenizer.vocabSize());
    std::printf("⭐ Chat template: %s\n", chatTemplateTypeName(gen_.type()));
    for (const std::string &s : stops_) std::printf("🛑 Stop: %s\n", s.c_str());
}

// n completions of one prompt (runChoices; n = 1 without `n`): the prompt is prefilled once. After one completion the cache
// keeps its answer too; after several, or after one cut at a stop string (its KV rows hold tokens past the cut), it keeps only the
// prompt messages, so a follow-up that quotes any one choice re-uses the prompt.
void ApiServer::complete(HttpRequest &req) {
    const ChatRequest chat = parseChat(req.json, cfg_, sampler_.vocabSize(), kMaxChoices);
    backend_.setLogprobs(chat.logprobs);   // refuses where they cannot run (tensor parallelism)
    sampler_.setControls(chat.presence, chat.frequency, chat.bias);
    sampler_.setFilters(chat.topK, chat.minP);
    sampler_.setTemperature(chat.temperature);
    sampler_.setTopp(chat.topp);
    if (chat.hasSeed) sampler_.setSeed(chat.seed);
    // several completions: choice i uses choiceSeed(base, i); without a seed the base is drawn from the advancing generator
    const uint64_t baseSeed = chat.hasSeed ? sampler_.seed() : (chat.n > 1 ? sampler_.nextSeed() : 0);
    const uint32_t seqLen = backend_.seqLen();
    const Prompt p = preparePrompt(gen_, tok_, cache_, chat.messages, seqLen, true);
    ChatResponse resp(req, chat, tok_, stops_, chat.n == 1);
    resp.start(p.publicPrompt);
    backend_.prefill(p.prefill, p.start);
    std::function<void(uint32_t, const TokenLogprobs &)> onLogprobs;
    if (chat.logprobs >= 0) onLogprobs = [&](uint32_t i, const TokenLogprobs &e) { resp.onLogprobs(i, e); };
    const std::vector<std::vector<int32_t>> out = runChoices(backend_, p.token, p.P, chat.n, chat.maxTokens, seqLen, sampler_, baseSeed,
                                                             [&](uint32_t i, int32_t t) { return resp.onToken(i, t); }, onLogprobs);
    if (chat.n == 1 && !resp.stopped(0)) rememberAnswer(cache_, p.P, out[0].size(), resp.text(0), seqLen);
    resp.finish(out, p.nPrompt);
    if (chat.n == 1) std::printf("🔶\n");
    else std::printf("(%u choices)🔶\n", chat.n);
}

void ApiServer::models(HttpRequest &req) const {
    req.writeJson("{\"object\": \"list\", \"data\": [{\"id\": " + jsonEscape(cfg_.modelName) + ", \"object\": \"model\", \"created\": 0, \"owned_by\": \"user\"}]}");
}

// ---- concurrent requests (--parallel): SlotScheduler (csrc/host/slot_scheduler.hpp) over SlotJobs ------------------------------

namespace {
// What the slots' requests share: the slots' prompt caches, the prompt tools and the connection count's close.
struct SlotServer {
    const ChatTemplateGenerator &gen;
    const Tokenizer &tok;
    std::vector<NaiveCache> caches;
    uint32_t slotLen;
    std::function<void(int)> close;   // closes a connection and counts it finished
};

// One validated chat completion: SlotScheduler's request, answered on its connection.
struct SlotJob {
    SlotServer &srv;
    HttpRequest req;
    ChatRequest chat;
    ChatResponse resp;
    uint32_t nPrompt = 0;
    std::map<std::pair<uint32_t, size_t>, uint32_t> promptLens;   // paged: P by (slot, cached messages), computed once
    SlotJob(SlotServer &s, HttpRequest r, ChatRequest c, const std::vector<std::string> &stops)
        : srv(s), req(std::move(r)), chat(std::move(c)), resp(req, chat, s.tok, stops) {}

    uint32_t n() const { return chat.n; }
    bool greedy() const { return chat.temperature == 0.f; }
    std::optional<uint64_t> seed() const { return chat.hasSeed ? std::optional<uint64_t>(chat.seed) : std::nullopt; }
    int64_t maxTokens() const { return chat.maxTokens; }
    int logprobs() const { return chat.logprobs; }
    size_t cachedPrefix(uint32_t slot) const { return srv.caches[slot].coveredPrefix(chat.messages); }
    uint32_t promptLen(uint32_t slot) {
        const auto key = std::make_pair(slot, cachedPrefix(slot));
        if (!promptLens.count(key)) { NaiveCache probe = srv.caches[slot]; promptLens[key] = preparePrompt(srv.gen, srv.tok, probe, chat.messages, srv.slotLen).P; }
        return promptLens[key];
    }
    SlotPrompt prepare(uint32_t slot) {
        const Prompt p = preparePrompt(srv.gen, srv.tok, srv.caches[slot], chat.messages, srv.slotLen);
        nPrompt = p.nPrompt;
        resp.start(p.publicPrompt);
        return p;
    }
    void onLogprobs(uint32_t i, const TokenLogprobs &e) { resp.onLogprobs(i, e); }
    bool onToken(uint32_t i, int32_t t) { return resp.onToken(i, t); }
    void finish(const std::vector<std::vector<int32_t>> &out, const std::vector<uint32_t> &slots, uint32_t P) {
        NaiveCache &cache = srv.caches[slots[0]];
        if (chat.n == 1 && !resp.stopped(0)) rememberAnswer(cache, P, out[0].size(), resp.text(0), srv.slotLen);
        for (size_t k = 1; k < slots.size(); k++) srv.caches[slots[k]].copyFrom(cache);   // they hold a copy of the prompt rows
        resp.finish(out, nPrompt);
        std::printf("🔶 slot %u%s\n", slots[0], chat.n > 1 ? (" (" + std::to_string(chat.n) + " choices)").c_str() : "");
        std::fflush(stdout);
        srv.close(req.fd);
    }
    void fail(std::exception_ptr error, const std::vector<uint32_t> &slots) {
        for (uint32_t s : slots) srv.caches[s].clear();   // their rows may not match what their caches say
        try {
            std::rethrow_exception(error);
        } catch (const std::exception &e) {
            std::printf("Socket error: %s\n", e.what());
        } catch (...) {
            std::printf("Socket error: unknown error\n");
        }
        std::fflush(stdout);
        srv.close(req.fd);
    }
};

// InferenceBackend's slot calls as SlotScheduler makes them.
struct SlotBackend {
    using Request = std::shared_ptr<SlotJob>;
    using Entry = TokenLogprobs;
    InferenceBackend &be;
    uint32_t slots() const { return be.slots(); }
    uint32_t slotLen() const { return be.slotLen(); }
    bool paged() const { return be.paged(); }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) { be.slotPrefill(slot, tokens, pos); }
    void slotCopy(uint32_t src, uint32_t dst, uint32_t P) { be.slotCopy(src, dst, P); }
    void slotSampling(uint32_t slot, uint64_t seed, const Request &r) {
        const ChatRequest &c = r->chat;
        be.slotSampling(slot, seed, c.temperature, c.topp, c.presence, c.frequency, c.bias);
        if (c.topK || c.minP > 0.f) be.slotFilters(slot, c.topK, c.minP);
    }
    void slotLogprobs(uint32_t slot, int k) { be.slotLogprobs(slot, k); }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &t, const std::vector<int32_t> &pos, uint32_t active) { return be.slotsStep(t, pos, active); }
    std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> &t, const std::vector<int32_t> &pos, uint32_t active, std::vector<Entry> &e) {
        return be.slotsStepLogprobs(t, pos, active, e);
    }
    bool slotReserve(uint32_t slot, uint32_t rows) { return be.slotReserve(slot, rows); }
    void slotTrim(uint32_t slot, uint32_t rows) { be.slotTrim(slot, rows); }
    void slotRelease(uint32_t slot) { be.slotRelease(slot); }
    uint32_t freePages() const { return be.freePages(); }
    uint32_t slotPageCount(uint32_t slot) const { return be.slotPageCount(slot); }
    template <class F> void asleep(const F &ready) const { while (!ready()) {} }
};
}  // namespace

void ApiServer::serveParallel(int srv) {
    std::mutex mu;
    std::condition_variable cv;
    int open = 0;   // connections accepted and not yet finished
    SlotServer slots{gen_, tok_, std::vector<NaiveCache>(cfg_.parallel), backend_.slotLen(), [&](int fd) {
        ::close(fd);
        std::lock_guard<std::mutex> lk(mu);
        open--;
        cv.notify_all();
    }};
    SlotScheduler<SlotBackend> sched(SlotBackend{backend_}, [this] { return sampler_.nextSeed(); }, [&](uint32_t s) { slots.caches[s].clear(); });
    // Reads and validates one connection; chat completions go to the engine thread, which closes them when they end.
    const auto handle = [&](int fd) {
        try {
            HttpRequest req = HttpRequest::read(fd);
            std::printf("🔷 %s %s\n", req.method.c_str(), req.path.c_str());
            std::fflush(stdout);
            if (req.method == "POST" && req.path == "/v1/chat/completions") {
                ChatRequest chat = parseChat(req.json, cfg_, sampler_.vocabSize(), cfg_.parallel);   // --parallel > 1 runs on one GPU
                sched.submit(std::make_shared<SlotJob>(slots, std::move(req), std::move(chat), stops_));
                return;
            }
            if (req.method == "OPTIONS") req.writeCors();
            else if (req.method == "GET" && req.path == "/v1/models") models(req);
            else req.writeNotFound();
        } catch (const std::exception &e) {
            std::printf("Socket error: %s\n", e.what());
            std::fflush(stdout);
        }
        slots.close(fd);
    };
    // Once it has served maxRequests connections and every one is finished, the engine thread stops.
    std::thread acceptor([&] {
        int one = 1, served = 0;
        while (cfg_.maxRequests == 0 || served < cfg_.maxRequests) {
            const int fd = ::accept(srv, nullptr, nullptr);
            if (fd < 0) continue;
            ::setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
            { std::lock_guard<std::mutex> lk(mu); open++; }
            std::thread(handle, fd).detach();
            served++;
        }
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return open == 0; });
        }
        sched.stop();
    });
    sched.run();
    acceptor.join();
    ::close(srv);
}

void ApiServer::serve() {
    const int srv = ::socket(AF_INET, SOCK_STREAM, 0);
    if (srv < 0) throw std::runtime_error("Cannot create socket");
    int one = 1;
    ::setsockopt(srv, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    sockaddr_in addr{};
    addr.sin_family = AF_INET;
    addr.sin_port = htons((uint16_t)cfg_.port);
    if (::inet_pton(AF_INET, cfg_.host.c_str(), &addr.sin_addr) != 1) { ::close(srv); throw std::runtime_error("Invalid host address: " + cfg_.host); }
    if (::bind(srv, (sockaddr *)&addr, sizeof(addr)) != 0 || ::listen(srv, 8) != 0) {
        ::close(srv);
        throw std::runtime_error("Cannot bind port " + std::to_string(cfg_.port));
    }
    if (cfg_.host == "0.0.0.0" || cfg_.host == "127.0.0.1") std::printf("Server URL: http://localhost:%d/v1/\n", cfg_.port);
    std::fflush(stdout);
    if (cfg_.parallel > 1) {
        if (backend_.slots() != cfg_.parallel) { ::close(srv); throw std::runtime_error("the backend has no KV-cache slots for --parallel"); }
        serveParallel(srv);
        return;
    }
    int served = 0;
    while (cfg_.maxRequests == 0 || served < cfg_.maxRequests) {
        const int fd = ::accept(srv, nullptr, nullptr);
        if (fd < 0) continue;
        ::setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
        try {
            HttpRequest req = HttpRequest::read(fd);
            std::printf("🔷 %s %s\n", req.method.c_str(), req.path.c_str());
            if (req.method == "OPTIONS") req.writeCors();
            else if (req.method == "POST" && req.path == "/v1/chat/completions") complete(req);
            else if (req.method == "GET" && req.path == "/v1/models") models(req);
            else req.writeNotFound();
        } catch (const std::exception &e) {
            std::printf("Socket error: %s\n", e.what());
        }
        std::fflush(stdout);
        ::close(fd);
        served++;
    }
    ::close(srv);
}

}  // namespace dl
