#include "model_format.hpp"

#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>

namespace dl {

const char *archName(ArchType a) {
    switch (a) {
        case ARCH_LLAMA: return "Llama";
        case ARCH_QWEN3: return "Qwen3";
        case ARCH_QWEN3_MOE: return "Qwen3 MoE";
    }
    throw std::runtime_error("Unsupported architecture");
}

const char *ropeName(RopeType r) {
    switch (r) {
        case ROPE_LLAMA: return "Llama";
        case ROPE_LLAMA3_1: return "Llama3.1";
        case ROPE_FALCON: return "Falcon";
    }
    throw std::runtime_error("Unsupported rope type");
}

static float epsilonFromCode(int32_t code) {
    if (code == 5) return 1e-5f;
    if (code == 6) return 1e-6f;
    throw std::runtime_error("Unsupported norm epsilon");
}

ModelHeader parseModelHeader(const uint8_t *data, size_t nBytes, uint64_t fileSize, uint32_t maxSeqLen) {
    if (nBytes < 8) throw std::runtime_error("Cannot read magic value");
    int32_t magic, headerSize;
    std::memcpy(&magic, data, 4);
    std::memcpy(&headerSize, data + 4, 4);
    if (magic == 0xABCD00 || magic == 0xABCD01) throw std::runtime_error("Old model format is not supported");
    if (magic != kModelMagic) throw std::runtime_error("Unsupported magic number");
    if (headerSize < 8 || (size_t)headerSize > nBytes || (headerSize - 8) % 8 != 0)
        throw std::runtime_error("Cannot read header values");

    ModelHeader h;
    h.headerSize = (uint64_t)headerSize;
    h.fileSize = fileSize;
    const int nPairs = (headerSize - 8) / 8;
    for (int i = 0; i < nPairs; i++) {
        int32_t key, value;
        std::memcpy(&key, data + 8 + 8 * i, 4);
        std::memcpy(&value, data + 12 + 8 * i, 4);
        switch (key) {
            case K_VERSION: h.version = value; break;
            case K_ARCH_TYPE: h.arch = (ArchType)value; break;
            case K_DIM: h.dim = value; break;
            case K_HIDDEN_DIM: h.hiddenDim = value; break;
            case K_N_LAYERS: h.nLayers = value; break;
            case K_N_HEADS: h.nHeads = value; break;
            case K_N_KV_HEADS: h.nKvHeads = value; break;
            case K_N_EXPERTS: h.nExperts = value; break;
            case K_N_ACTIVE_EXPERTS: h.nActiveExperts = value; break;
            case K_VOCAB_SIZE: h.vocabSize = value; break;
            case K_SEQ_LEN: h.seqLen = value; break;
            case K_HIDDEN_ACT: h.hiddenAct = (HiddenAct)value; break;
            case K_ROPE_THETA: h.ropeTheta = (float)value; break;
            case K_WEIGHT_FLOAT_TYPE: h.weightType = (FloatType)value; break;
            case K_ROPE_SCALING_FACTOR: h.ropeScalingFactor = (float)value; break;
            case K_ROPE_SCALING_LOW_FREQ_FACTOR: h.ropeScalingLowFreqFactor = (float)value; break;
            case K_ROPE_SCALING_HIGH_FREQ_FACTOR: h.ropeScalingHighFreqFactor = (float)value; break;
            case K_ROPE_SCALING_ORIG_MAX_SEQ_LEN: h.ropeScalingOrigMaxSeqLen = value; break;
            case K_ROPE_TYPE: h.ropeType = (RopeType)value; break;
            case K_HEAD_DIM: h.headDim = value; break;
            case K_NORM_EPSILON: h.normEpsilon = epsilonFromCode(value); break;
            case K_MOE_HIDDEN_DIM: h.moeHiddenDim = value; break;
            default: throw std::runtime_error("Unsupported header key");
        }
    }
    if (h.weightType == F_UNK) throw std::runtime_error("Model does not specify weight type");
    if (h.arch != ARCH_LLAMA && h.arch != ARCH_QWEN3 && h.arch != ARCH_QWEN3_MOE)
        throw std::runtime_error("Unsupported architecture");
    if (h.dim == 0 || h.nHeads == 0 || h.nKvHeads == 0 || h.nLayers == 0 || h.vocabSize == 0)
        throw std::runtime_error("Model header is incomplete");

    h.origSeqLen = h.seqLen;
    if (maxSeqLen > 0 && h.seqLen > maxSeqLen) h.seqLen = maxSeqLen;
    if (h.headDim == 0) h.headDim = h.dim / h.nHeads;
    h.qDim = h.headDim * h.nHeads;
    h.kvDim = h.headDim * h.nKvHeads;
    if (h.qkNorm()) h.ropeType = ROPE_FALCON;  // Qwen3 checkpoints keep the half-split (NeoX) layout
    return h;
}

ModelHeader loadModelHeader(const std::string &path, uint32_t maxSeqLen) {
    std::unique_ptr<FILE, int (*)(FILE *)> f(std::fopen(path.c_str(), "rb"), std::fclose);
    if (!f) throw std::runtime_error("Cannot open model file (" + path + "): " + std::strerror(errno));
    uint8_t head[8];
    if (std::fread(head, 1, 8, f.get()) != 8) throw std::runtime_error("Cannot read magic value");
    int32_t magic, headerSize;
    std::memcpy(&magic, head, 4);
    std::memcpy(&headerSize, head + 4, 4);
    if (magic == 0xABCD00 || magic == 0xABCD01) throw std::runtime_error("Old model format is not supported");
    if (magic != kModelMagic) throw std::runtime_error("Unsupported magic number");
    if (headerSize < 8 || headerSize > (1 << 20)) throw std::runtime_error("Cannot read header size");
    std::vector<uint8_t> buf(headerSize);
    std::memcpy(buf.data(), head, 8);
    if (headerSize > 8 && std::fread(buf.data() + 8, 1, headerSize - 8, f.get()) != (size_t)headerSize - 8)
        throw std::runtime_error("Cannot read header values");
    std::fseek(f.get(), 0, SEEK_END);
    const uint64_t fileSize = (uint64_t)ftello(f.get());
    return parseModelHeader(buf.data(), buf.size(), fileSize, maxSeqLen);
}

std::vector<uint8_t> buildModelHeader(const std::vector<std::pair<int32_t, int32_t>> &kv) {
    std::vector<uint8_t> out(8 + 8 * kv.size());
    const int32_t magic = kModelMagic, size = (int32_t)out.size();
    std::memcpy(out.data(), &magic, 4);
    std::memcpy(out.data() + 4, &size, 4);
    for (size_t i = 0; i < kv.size(); i++) {
        std::memcpy(out.data() + 8 + 8 * i, &kv[i].first, 4);
        std::memcpy(out.data() + 12 + 8 * i, &kv[i].second, 4);
    }
    return out;
}

std::string describeModelHeader(const ModelHeader &h) {
    char line[256];
    std::string s;
    auto add = [&](const char *fmt, auto... a) { std::snprintf(line, sizeof(line), fmt, a...); s += line; };
    add("💡 Arch: %s\n", archName(h.arch));
    add("💡 HiddenAct: %s\n", h.hiddenAct == ACT_GELU ? "Gelu" : "Silu");
    add("💡 Dim: %u\n", h.dim);
    add("💡 HeadDim: %u\n", h.headDim);
    add("💡 QDim: %u\n", h.qDim);
    add("💡 KvDim: %u\n", h.kvDim);
    add("💡 HiddenDim: %u\n", h.hiddenDim);
    add("💡 VocabSize: %u\n", h.vocabSize);
    add("💡 nLayers: %u\n", h.nLayers);
    add("💡 nHeads: %u\n", h.nHeads);
    add("💡 nKvHeads: %u\n", h.nKvHeads);
    if (h.seqLen != h.origSeqLen) add("💡 OrigSeqLen: %u\n", h.origSeqLen);
    if (h.nExperts > 0) {
        add("💡 nExperts: %u\n", h.nExperts);
        add("💡 nActiveExperts: %u\n", h.nActiveExperts);
        add("💡 MoeHiddenDim: %u\n", h.moeHiddenDim);
    }
    add("💡 SeqLen: %u\n", h.seqLen);
    add("💡 NormEpsilon: %f\n", h.normEpsilon);
    add("💡 RopeType: %s\n", ropeName(h.ropeType));
    add("💡 RopeTheta: %.0f\n", h.ropeTheta);
    if (h.ropeType == ROPE_LLAMA3_1)
        add("💡 RopeScaling: f=%.1f, l=%.1f, h=%.1f, o=%d\n", h.ropeScalingFactor, h.ropeScalingLowFreqFactor,
            h.ropeScalingHighFreqFactor, (int)h.ropeScalingOrigMaxSeqLen);
    return s;
}

// ---- tensor directory ---------------------------------------------------------------------------

std::vector<TensorEntry> buildTensorDirectory(const ModelHeader &h, bool checkFileSize) {
    std::vector<TensorEntry> dir;
    uint64_t cursor = h.headerSize;
    auto add = [&](const char *name, uint32_t layer, uint32_t expert, FloatType type, uint64_t d, uint64_t n, Partition part) {
        TensorEntry t;
        t.name = name; t.layer = layer; t.expert = expert; t.type = type; t.d = d; t.n = n; t.part = part;
        t.offset = cursor;
        t.nBytes = tensorBytes(type, d * n);
        cursor += t.nBytes;
        dir.push_back(std::move(t));
    };
    const FloatType w = h.weightType;
    const uint64_t ff = h.ffDim();
    add("embedding", 0, 0, F_32, h.vocabSize, h.dim, PART_ROOT);
    for (uint32_t l = 0; l < h.nLayers; l++) {
        add("block_matmul_q", l, 0, w, h.qDim, h.dim, PART_ROWS);
        add("block_matmul_k", l, 0, w, h.kvDim, h.dim, PART_ROWS);
        add("block_matmul_v", l, 0, w, h.kvDim, h.dim, PART_ROWS);
        add("block_matmul_wo", l, 0, w, h.dim, h.qDim, PART_COLS);
        if (h.nExperts > 0) {
            add("block_moe_gate", l, 0, F_32, h.nExperts, h.dim, PART_REPLICATE);
            for (uint32_t e = 0; e < h.nExperts; e++) {
                add("block_matmul_w1", l, e, w, ff, h.dim, PART_ROWS);
                add("block_matmul_w2", l, e, w, h.dim, ff, PART_COLS);
                add("block_matmul_w3", l, e, w, ff, h.dim, PART_ROWS);
            }
        } else {
            add("block_matmul_w1", l, 0, w, ff, h.dim, PART_ROWS);
            add("block_matmul_w2", l, 0, w, h.dim, ff, PART_COLS);
            add("block_matmul_w3", l, 0, w, ff, h.dim, PART_ROWS);
        }
        if (h.qkNorm()) {
            add("block_norm_q", l, 0, F_32, 1, h.headDim, PART_REPLICATE);
            add("block_norm_k", l, 0, F_32, 1, h.headDim, PART_REPLICATE);
        }
        add("block_norm_0", l, 0, F_32, 1, h.dim, PART_REPLICATE);
        add("block_norm_1", l, 0, F_32, 1, h.dim, PART_REPLICATE);
    }
    add("final_norm", 0, 0, F_32, 1, h.dim, PART_REPLICATE);
    add("final_matmul_logits", 0, 0, w, h.vocabSize, h.dim, PART_ROWS);
    if (checkFileSize && cursor != h.fileSize)
        throw std::runtime_error("Missing bytes in weight file: " + std::to_string((long long)cursor - (long long)h.fileSize));
    return dir;
}

SliceRange sliceTensor(const TensorEntry &t, uint32_t rank, uint32_t nRanks) {
    if (nRanks == 0 || rank >= nRanks) throw std::invalid_argument("bad rank");
    SliceRange s;
    const uint64_t blk = blockElems(t.type);
    s.rowBytes = tensorBytes(t.type, t.n);
    s.firstRow = 0; s.nRows = t.d;
    s.firstCol = 0; s.nCols = t.n;
    if (t.part == PART_ROWS) {
        if (t.d % nRanks) throw std::invalid_argument(t.name + ": rows not divisible by the number of ranks");
        s.nRows = t.d / nRanks;
        s.firstRow = s.nRows * rank;
    } else if (t.part == PART_COLS) {
        if (t.n % nRanks || (t.n / nRanks) % blk)
            throw std::invalid_argument(t.name + ": columns not divisible into whole quant blocks per rank");
        s.nCols = t.n / nRanks;
        s.firstCol = s.nCols * rank;
    }
    s.colByteOffset = tensorBytes(t.type, s.firstCol);
    s.colBytes = tensorBytes(t.type, s.nCols);
    return s;
}

uint64_t extractSlice(const TensorEntry &t, const uint8_t *fileBase, uint32_t rank, uint32_t nRanks, uint8_t *out) {
    const SliceRange s = sliceTensor(t, rank, nRanks);
    const uint8_t *src = fileBase + t.offset + s.firstRow * s.rowBytes + s.colByteOffset;
    if (s.colBytes == s.rowBytes) {
        std::memcpy(out, src, s.nRows * s.rowBytes);
    } else {
        for (uint64_t r = 0; r < s.nRows; r++) std::memcpy(out + r * s.colBytes, src + r * s.rowBytes, s.colBytes);
    }
    return s.totalBytes();
}

// ---- RoPE ---------------------------------------------------------------------------------------

float ropeFrequency(const ModelHeader &h, uint32_t j) {
    const float hd = (float)h.headDim;
    float freq = 1.0f / std::pow(h.ropeTheta, (float)(2 * j) / hd);
    if (h.ropeType == ROPE_LLAMA3_1 && h.ropeScalingFactor != 1.0f) {
        const float twoPi = 6.28318530717958647692f;
        const float waveLen = twoPi / freq;
        const float orig = (float)h.ropeScalingOrigMaxSeqLen;
        const float highWave = orig / h.ropeScalingHighFreqFactor;
        const float lowWave = orig / h.ropeScalingLowFreqFactor;
        if (waveLen < highWave) {
            // unchanged
        } else if (waveLen > lowWave) {
            freq = freq / h.ropeScalingFactor;
        } else {
            const float smooth = (orig / waveLen - h.ropeScalingLowFreqFactor) /
                                 (h.ropeScalingHighFreqFactor - h.ropeScalingLowFreqFactor);
            freq = (1.f - smooth) * freq / h.ropeScalingFactor + smooth * freq;
        }
    }
    return freq;
}

void buildRopeTable(const ModelHeader &h, uint32_t seqLen, float *out) {
    const uint32_t half = h.headDim / 2;
    std::vector<float> freq(half);
    for (uint32_t j = 0; j < half; j++) freq[j] = ropeFrequency(h, j);
    for (uint32_t pos = 0; pos < seqLen; pos++) {
        for (uint32_t j = 0; j < half; j++) {
            const float a = (float)pos * freq[j];
            out[((uint64_t)pos * half + j) * 2 + 0] = std::cos(a);
            out[((uint64_t)pos * half + j) * 2 + 1] = std::sin(a);
        }
    }
}

uint64_t requiredDeviceBytes(const ModelHeader &h, uint32_t nRanks, uint32_t kvBytesPerElem) {
    uint64_t total = 0;
    for (const TensorEntry &t : buildTensorDirectory(h, false)) {
        // device size: q40 keeps its blocks, f16 / f32 stay as they are, q80 matrices are dequantised to f32 (models/loader.py)
        const uint64_t bytes = t.type == F_Q80 ? t.d * t.n * 4 : t.nBytes;
        if (t.part == PART_ROOT || t.part == PART_REPLICATE) total += bytes;
        else total += bytes / nRanks;
    }
    const uint64_t kvHeads = h.nKvHeads >= nRanks ? h.nKvHeads / nRanks : 1;
    total += (uint64_t)2 * h.nLayers * h.seqLen * kvHeads * h.headDim * kvBytesPerElem;
    return total;
}

}  // namespace dl
