// Minimal JSON reader/writer for the API server (the reference vendors nlohmann/json, 24 kLoC; the server only needs objects,
// arrays, strings with escapes, numbers, booleans and null on input, and string escaping on output).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

namespace dl {

struct JsonValue {
    enum Kind { Null, Bool, Number, String, Array, Object } kind = Null;
    bool b = false;
    double num = 0;
    bool integral = false;   // Number written without a fraction or exponent (`1`, not `1.0`)
    bool loneSurrogate = false;   // String with a \u escape of an unpaired surrogate (stored as U+FFFD)
    std::string str;
    std::vector<JsonValue> arr;
    std::vector<std::pair<std::string, JsonValue>> obj;   // insertion order kept

    bool isObject() const { return kind == Object; }
    bool isArray() const { return kind == Array; }
    bool isString() const { return kind == String; }
    const JsonValue *find(const std::string &key) const {
        if (kind != Object) return nullptr;
        for (const auto &kv : obj) if (kv.first == key) return &kv.second;
        return nullptr;
    }
    const JsonValue &at(const std::string &key) const {
        const JsonValue *v = find(key);
        if (!v) throw std::runtime_error("JSON: missing key \"" + key + "\"");
        return *v;
    }
    double numberOr(const std::string &key, double dflt) const {
        const JsonValue *v = find(key);
        return (v && v->kind == Number) ? v->num : dflt;
    }
    bool boolOr(const std::string &key, bool dflt) const {
        const JsonValue *v = find(key);
        return (v && v->kind == Bool) ? v->b : dflt;
    }
};

class JsonParser {
public:
    explicit JsonParser(const std::string &text) : s_(text) {}
    JsonValue parse() {
        JsonValue v = value();
        ws();
        if (p_ != s_.size()) fail("trailing characters");
        return v;
    }

private:
    const std::string &s_;
    size_t p_ = 0;
    [[noreturn]] void fail(const char *what) const { throw std::runtime_error(std::string("JSON parse error: ") + what + " at offset " + std::to_string(p_)); }
    void ws() { while (p_ < s_.size() && (s_[p_] == ' ' || s_[p_] == '\n' || s_[p_] == '\r' || s_[p_] == '\t')) p_++; }
    bool eat(const char *lit) {
        size_t n = 0;
        while (lit[n]) n++;
        if (s_.compare(p_, n, lit) == 0) { p_ += n; return true; }
        return false;
    }
    static void utf8(std::string &out, uint32_t cp) {
        if (cp < 0x80) out += (char)cp;
        else if (cp < 0x800) { out += (char)(0xC0 | (cp >> 6)); out += (char)(0x80 | (cp & 0x3F)); }
        else if (cp < 0x10000) { out += (char)(0xE0 | (cp >> 12)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
        else { out += (char)(0xF0 | (cp >> 18)); out += (char)(0x80 | ((cp >> 12) & 0x3F)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
    }
    uint32_t hex4() {
        if (p_ + 4 > s_.size()) fail("bad \\u escape");
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) {
            const char c = s_[p_++];
            v <<= 4;
            if (c >= '0' && c <= '9') v |= (uint32_t)(c - '0');
            else if (c >= 'a' && c <= 'f') v |= (uint32_t)(c - 'a' + 10);
            else if (c >= 'A' && c <= 'F') v |= (uint32_t)(c - 'A' + 10);
            else fail("bad \\u escape");
        }
        return v;
    }
    std::string string(bool *loneSurrogate = nullptr) {
        if (s_[p_] != '"') fail("expected string");
        p_++;
        std::string out;
        while (true) {
            if (p_ >= s_.size()) fail("unterminated string");
            const char c = s_[p_++];
            if (c == '"') break;
            if (c != '\\') { out += c; continue; }
            if (p_ >= s_.size()) fail("bad escape");
            const char e = s_[p_++];
            switch (e) {
                case '"': out += '"'; break;
                case '\\': out += '\\'; break;
                case '/': out += '/'; break;
                case 'b': out += '\b'; break;
                case 'f': out += '\f'; break;
                case 'n': out += '\n'; break;
                case 'r': out += '\r'; break;
                case 't': out += '\t'; break;
                case 'u': {
                    uint32_t cp = hex4();
                    if (cp >= 0xD800 && cp <= 0xDBFF && p_ + 1 < s_.size() && s_[p_] == '\\' && s_[p_ + 1] == 'u') {
                        p_ += 2;
                        const uint32_t lo = hex4();
                        if (lo >= 0xDC00 && lo <= 0xDFFF) cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                        else {
                            utf8(out, 0xFFFD);
                            if (loneSurrogate) *loneSurrogate = true;
                            cp = lo;
                        }
                    }
                    if (cp >= 0xD800 && cp <= 0xDFFF) {   // unpaired surrogate
                        cp = 0xFFFD;
                        if (loneSurrogate) *loneSurrogate = true;
                    }
                    utf8(out, cp);
                    break;
                }
                default: fail("bad escape");
            }
        }
        return out;
    }
    JsonValue value() {
        ws();
        if (p_ >= s_.size()) fail("unexpected end");
        JsonValue v;
        const char c = s_[p_];
        if (c == '{') {
            v.kind = JsonValue::Object;
            p_++;
            ws();
            if (p_ < s_.size() && s_[p_] == '}') { p_++; return v; }
            while (true) {
                ws();
                std::string key = string();
                ws();
                if (p_ >= s_.size() || s_[p_] != ':') fail("expected ':'");
                p_++;
                v.obj.emplace_back(std::move(key), value());
                ws();
                if (p_ < s_.size() && s_[p_] == ',') { p_++; continue; }
                if (p_ < s_.size() && s_[p_] == '}') { p_++; break; }
                fail("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.kind = JsonValue::Array;
            p_++;
            ws();
            if (p_ < s_.size() && s_[p_] == ']') { p_++; return v; }
            while (true) {
                v.arr.push_back(value());
                ws();
                if (p_ < s_.size() && s_[p_] == ',') { p_++; continue; }
                if (p_ < s_.size() && s_[p_] == ']') { p_++; break; }
                fail("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.kind = JsonValue::String;
            v.str = string(&v.loneSurrogate);
        } else if (eat("true")) { v.kind = JsonValue::Bool; v.b = true; }
        else if (eat("false")) { v.kind = JsonValue::Bool; v.b = false; }
        else if (eat("null")) { v.kind = JsonValue::Null; }
        else {
            const char *start = s_.c_str() + p_;
            char *end = nullptr;
            v.num = std::strtod(start, &end);
            if (end == start) fail("unexpected character");
            v.kind = JsonValue::Number;
            v.integral = std::string(start, (size_t)(end - start)).find_first_of(".eE") == std::string::npos;
            p_ += (size_t)(end - start);
        }
        return v;
    }
};

inline std::string jsonEscape(const std::string &s) {
    std::string out = "\"";
    for (unsigned char c : s) {
        switch (c) {
            case '"': out += "\\\""; break;
            case '\\': out += "\\\\"; break;
            case '\n': out += "\\n"; break;
            case '\r': out += "\\r"; break;
            case '\t': out += "\\t"; break;
            case '\b': out += "\\b"; break;
            case '\f': out += "\\f"; break;
            default:
                if (c < 0x20) { char buf[8]; std::snprintf(buf, sizeof(buf), "\\u%04x", c); out += buf; }
                else out += (char)c;
        }
    }
    out += '"';
    return out;
}

}  // namespace dl
