#include "api_server.hpp"

#include <arpa/inet.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/socket.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <ctime>
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

std::string chunkJson(const std::string *delta, bool stop, uint32_t index) {
    std::string s = "{\"id\": \"cmpl-c0\", \"object\": \"chat.completion\", \"created\": " + std::to_string((long long)std::time(nullptr)) +
                    ", \"model\": \"Distributed Model\", \"choices\": [{\"index\": " + std::to_string(index) + ", \"finish_reason\": " +
                    (stop ? "\"stop\"" : "\"\"");
    if (!stop) s += ", \"delta\": {\"role\": \"assistant\", \"content\": " + jsonEscape(delta ? *delta : std::string()) + "}";
    s += "}]}";
    return s;
}

// ---- several completions of one prompt ------------------------------------------------------------------------------------

std::vector<std::vector<int32_t>> runChoices(InferenceBackend &backend, int32_t token, uint32_t P, uint32_t n, int maxTokens, uint32_t seqLen,
                                             Sampler &sampler, uint64_t baseSeed, const std::function<bool(uint32_t, int32_t)> &onToken) {
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
        while (out[first].size() < limit) {
            tok = backend.next(tok, pos++, smp);
            for (uint32_t i = first; i <= last; i++) {
                if (done[i]) continue;
                out[i].push_back(tok);
                if (onToken(i, tok)) { done[i] = true; nDone++; }
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
        for (uint32_t i = 0; i < n; i++) {
            if (!((active >> i) & 1u)) continue;
            out[i].push_back(last[i]);
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

float parsePenalty(const std::string &flag, const std::string &value) {
    const float v = std::stof(value);
    if (!(v >= -kMaxPenalty && v <= kMaxPenalty)) throw std::runtime_error(flag + " must be from -2 to 2");
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
// keeps its answer too; after several it keeps only the prompt messages, so a follow-up that quotes any one choice re-uses the
// prompt.
void ApiServer::complete(HttpRequest &req) {
    if (!req.hasJson || !req.json.isObject()) throw std::runtime_error("request body must be a JSON object");
    const JsonValue &body = req.json;
    std::vector<ChatItem> messages;
    for (const JsonValue &m : body.at("messages").arr) messages.push_back({m.at("role").str, m.at("content").str});
    const bool stream = body.boolOr("stream", false);
    const int maxTokens = (int)body.numberOr("max_tokens", -1);
    sampler_.setTemperature((float)body.numberOr("temperature", cfg_.temperature));
    sampler_.setTopp((float)body.numberOr("top_p", cfg_.topp));
    uint32_t n = 1;
    if (const JsonValue *v = body.find("n")) {
        if (v->kind != JsonValue::Number || v->num != (double)(int64_t)v->num || v->num < 1 || v->num > kMaxChoices)
            throw std::runtime_error("'n' must be an integer from 1 to 8");
        n = (uint32_t)v->num;
    }
    float presence = cfg_.presencePenalty, frequency = cfg_.frequencyPenalty;
    std::vector<std::pair<int32_t, float>> bias;
    parseControls(body, sampler_.vocabSize(), presence, frequency, bias);
    sampler_.setControls(presence, frequency, bias);
    bool seeded = false;
    if (const JsonValue *s = body.find("seed")) if (s->kind == JsonValue::Number) { sampler_.setSeed((uint64_t)s->num); seeded = true; }
    // several completions: choice i uses choiceSeed(base, i); without a seed the base is drawn from the advancing generator
    const uint64_t baseSeed = seeded ? sampler_.seed() : (n > 1 ? sampler_.nextSeed() : 0);

    const uint32_t seqLen = backend_.seqLen();
    const uint32_t startPos = cache_.resolveDeltaPrompt(messages);
    const GeneratedChat g = gen_.generate(messages, true);
    std::printf("🔹%s🔸", g.content.c_str());
    const std::vector<int32_t> tokens = tok_.encode(g.content, startPos == 0, true);
    const uint32_t nPrompt = (uint32_t)tokens.size();
    const uint32_t promptEnd = std::min(startPos + nPrompt - 1, seqLen);
    for (const ChatItem &m : messages) cache_.push(promptEnd, m);

    std::vector<EosDetector> dets(n, EosDetector(tok_.data().eosIds, stops_, maxLen(stops_), maxLen(stops_)));
    std::vector<std::string> pending(n), buffers(n, g.publicPrompt);
    if (stream) {
        req.writeStreamStart();
        if (!g.publicPrompt.empty())
            for (uint32_t i = 0; i < n; i++) req.writeStreamChunk("data: " + chunkJson(&g.publicPrompt, false, i) + "\r\n\r\n");
    }
    const uint32_t nPref = promptEnd - startPos;
    backend_.prefill(std::vector<int32_t>(tokens.begin(), tokens.begin() + nPref), startPos);
    const int32_t token = nPref < tokens.size() ? tokens[nPref] : tokens.back();
    const auto onToken = [&](uint32_t i, int32_t t) {
        const std::string piece = tok_.decodeWith(pending[i], t);
        if (n == 1 && !piece.empty()) { std::printf("%s", piece.c_str()); std::fflush(stdout); }
        const EosDetectorResult kind = dets[i].append(t, piece);
        if (kind == NOT_EOS || kind == EOS) {
            const std::string delta = dets[i].getDelta();
            if (!delta.empty()) {
                if (stream) req.writeStreamChunk("data: " + chunkJson(&delta, false, i) + "\r\n\r\n");
                buffers[i] += delta;
            }
            dets[i].reset();
        }
        return kind == EOS;
    };
    const std::vector<std::vector<int32_t>> out = runChoices(backend_, token, promptEnd, n, maxTokens, seqLen, sampler_, baseSeed, onToken);
    if (n == 1) {
        const uint32_t end = promptEnd + (uint32_t)out[0].size();
        if (end == seqLen) cache_.clear();
        else cache_.push(end, {"assistant", buffers[0]});
    }
    if (stream) {
        for (uint32_t i = 0; i < n; i++) req.writeStreamChunk("data: " + chunkJson(nullptr, true, i) + "\r\n\r\n");
        req.writeStreamChunk("data: [DONE]");
        req.writeStreamEnd();
    } else {
        uint32_t nCompletion = 0;
        std::string choices;
        for (uint32_t i = 0; i < n; i++) {
            nCompletion += (uint32_t)out[i].size();
            choices += std::string(i ? ", " : "") + "{\"index\": " + std::to_string(i) + ", \"message\": {\"role\": \"assistant\", \"content\": " +
                       jsonEscape(buffers[i]) + "}, \"finish_reason\": \"stop\"}";
        }
        req.writeJson("{\"id\": \"cmpl-j0\", \"object\": \"chat.completion\", \"created\": " + std::to_string((long long)std::time(nullptr)) +
                      ", \"model\": \"Distributed Model\", \"usage\": {\"completion_tokens\": " + std::to_string(nCompletion) +
                      ", \"prompt_tokens\": " + std::to_string(nPrompt) + ", \"total_tokens\": " + std::to_string(nPrompt + nCompletion) +
                      "}, \"choices\": [" + choices + "]}");
    }
    if (n == 1) std::printf("🔶\n");
    else std::printf("(%u choices)🔶\n", n);
}

void ApiServer::models(HttpRequest &req) const {
    req.writeJson("{\"object\": \"list\", \"data\": [{\"id\": " + jsonEscape(cfg_.modelName) + ", \"object\": \"model\", \"created\": 0, \"owned_by\": \"user\"}]}");
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
