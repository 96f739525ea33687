#include "native_engine.hpp"

#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <stdexcept>
#include <tuple>

#include "../cuda/engine_api.h"

namespace dl {

namespace {

void cudaCheck(cudaError_t e, const char *what) {
    if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
void engCheck(int rc, const char *what) {
    if (rc != 0) throw std::runtime_error(std::string(what) + " failed with code " + std::to_string(rc));
}

struct Mapping {   // read-only mmap of the model file
    const uint8_t *data = nullptr;
    size_t size = 0;
    explicit Mapping(const std::string &path) {
        const int fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) throw std::runtime_error("Cannot open model file: " + path);
        struct stat st {};
        if (::fstat(fd, &st) != 0) { ::close(fd); throw std::runtime_error("Cannot stat model file: " + path); }
        size = (size_t)st.st_size;
        void *p = ::mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
        ::close(fd);
        if (p == MAP_FAILED) throw std::runtime_error("Cannot mmap model file: " + path);
        data = (const uint8_t *)p;
    }
    ~Mapping() { if (data) ::munmap((void *)data, size); }
};

struct Q40Dev {   // device layout of csrc/cuda/common.cuh: qs u32 [rows][n/8], scales f16 [rows][n/32]
    void *qs = nullptr, *scales = nullptr;
};

}  // namespace

struct NativeEngine::Impl {
    std::vector<void *> allocations;
    void *engine = nullptr;
    void *vmm = nullptr;               // peer-memory arena handle (tensor parallel)
    cudaStream_t stream = nullptr;
    // weights
    float *embedding = nullptr, *finalNorm = nullptr, *rope = nullptr;
    Q40Dev wcls;
    struct Layer {
        Q40Dev qkv, wo, w13, w2;
        float *norm0 = nullptr, *norm1 = nullptr, *qNorm = nullptr, *kNorm = nullptr, *moeGate = nullptr;
        void *kCache = nullptr, *vCache = nullptr;
        void *kScale = nullptr, *vScale = nullptr;   // q80 cache (kvType 1)
    };
    std::vector<Layer> layers;
    // activations / state
    int32_t *tokens = nullptr, *pos = nullptr, *history = nullptr;
    float *logits = nullptr;
    std::vector<float> hostLogits;
    std::map<std::tuple<std::string, uint32_t, uint32_t>, const TensorEntry *> index;
    const TensorEntry &entry(const std::string &name, uint32_t layer = 0, uint32_t expert = 0) const {
        auto it = index.find(std::make_tuple(name, layer, expert));
        if (it == index.end()) throw std::runtime_error("tensor not found in the model file: " + name);
        return *it->second;
    }
};

void *NativeEngine::dev(size_t bytes) {
    void *p = nullptr;
    if (bytes == 0) bytes = 16;
    cudaCheck(cudaMalloc(&p, bytes), "cudaMalloc");
    impl_->allocations.push_back(p);
    cudaCheck(cudaMemsetAsync(p, 0, bytes, impl_->stream), "cudaMemset");   // every later write to p is ordered on the same stream
    return p;
}

NativeEngine::NativeEngine(const std::string &modelPath, uint32_t maxSeqLen, int device, uint32_t rank, uint32_t nRanks,
                           const std::string &commTag, std::function<void()> hostBarrier, uint32_t kvType) {
    rank_ = rank; nRanks_ = std::max(1u, nRanks);
    h_ = loadModelHeader(modelPath, maxSeqLen);
    if (h_.weightType != F_Q40)
        throw std::runtime_error("dllama-native runs q40 weight files; f32/f16/q80 files are served by the Python front end (./dllama)");
    if (h_.headDim != 64 && h_.headDim != 128) throw std::runtime_error("unsupported head dimension");
    dir_ = buildTensorDirectory(h_, true);
    seqLen_ = h_.seqLen;
    if (kvType > 1) throw std::runtime_error("unknown KV-cache float type");
    kvType_ = kvType;
    impl_ = new Impl();
    try {
        cudaCheck(cudaSetDevice(device), "cudaSetDevice");
        cudaCheck(cudaStreamCreateWithFlags(&impl_->stream, cudaStreamNonBlocking), "cudaStreamCreate");
        for (const TensorEntry &t : dir_) impl_->index[std::make_tuple(t.name, t.layer, t.expert)] = &t;
        int sms = 0;
        cudaCheck(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device), "cudaDeviceGetAttribute");
        const uint32_t hd = h_.headDim, dim = h_.dim, vocab = h_.vocabSize, N = nRanks_;
        // tensor-parallel placement (same rules as distributed_llama_b200/models/loader.py; reference slicers src/nn/nn-core.cpp:223-322):
        // more ranks than KV heads -> nRanks / nKvHeads ranks share one KV head, each with its own query heads of that group
        uint32_t kvRep = 1;
        if (N > h_.nKvHeads) {
            if (N % h_.nKvHeads || (h_.nHeads / h_.nKvHeads) % (N / h_.nKvHeads))
                throw std::runtime_error("the number of GPUs must be a multiple of nKvHeads that divides the query heads of a KV group");
            kvRep = N / h_.nKvHeads;
        }
        if (h_.nHeads % N || (kvRep == 1 && h_.nKvHeads % N) || h_.ffDim() % N || vocab % N)
            throw std::runtime_error("nHeads, nKvHeads, ffDim and vocabSize must be divisible by the number of GPUs");
        headsL_ = h_.nHeads / N; kvHeadsL_ = kvRep > 1 ? 1 : h_.nKvHeads / N;
        kvRank_ = rank_ / kvRep; kvSlices_ = N / kvRep;
        ffL_ = h_.ffDim() / N; vocabL_ = vocab / N;
        const uint32_t ff = ffL_;
        const uint32_t qDim = headsL_ * hd, kvDim = kvHeadsL_ * hd;
        if (N > 1 && (qDim % 128 || ff % 128))
            throw std::runtime_error("per-GPU slices of WO / W2 must be multiples of 128 columns (use fewer GPUs)");
        qkvDim_ = qDim + 2 * kvDim;
        const bool moe = h_.nExperts > 0;
        maxBatch_ = moe ? 1 : 8;
        nSplits_ = (uint32_t)std::max(1, std::min(32, (2 * sms) / (int)std::max(1u, headsL_)));

        Mapping file(modelPath);
        uploadWeights(file.data);

        // ---- the buffers this class reads or writes (the engine allocates its scratch itself) ----
        Impl &I = *impl_;
        const uint32_t mb = maxBatch_;
        I.tokens = (int32_t *)dev(mb * 4); I.pos = (int32_t *)dev(mb * 4);
        I.logits = (float *)dev((size_t)mb * vocabL_ * 4);
        I.hostLogits.resize(vocab);
        I.history = (int32_t *)dev((size_t)(seqLen_ + 1) * 4);
        GlobalPtrs g{};
        g.embedding = I.embedding; g.finalNorm = I.finalNorm; g.wclsQs = I.wcls.qs; g.wclsSc = I.wcls.scales; g.rope = I.rope;
        g.vocabFull = vocab; g.tokens = I.tokens; g.pos = I.pos; g.x = (float *)dev((size_t)mb * dim * 4); g.logits = I.logits;
        g.history = I.history;

        EngineConfig cfg{};
        cfg.dim = dim; cfg.nLayers = h_.nLayers; cfg.nHeads = headsL_; cfg.nKvHeads = kvHeadsL_; cfg.headDim = hd; cfg.ffDim = ff;
        cfg.vocab = vocabL_; cfg.seqLen = seqLen_; cfg.nExperts = h_.nExperts; cfg.nActiveExperts = h_.nActiveExperts; cfg.maxBatch = mb;
        cfg.nSplits = nSplits_; cfg.rank = rank_; cfg.nRanks = N; cfg.numSms = (uint32_t)sms; cfg.eps = h_.normEpsilon; cfg.usePdl = 1;
        cfg.moeFirstExpert = 0; cfg.moeNumLocal = h_.nExperts; cfg.wType = 0;
        cfg.hiddenAct = h_.hiddenAct == ACT_GELU ? 1u : 0u;
        cfg.kvType = kvType_;
        cfg.maxPrefill = 192;
        I.engine = dl_engine_create(&cfg);
        if (!I.engine) throw std::runtime_error("dl_engine_create failed");
        for (uint32_t l = 0; l < h_.nLayers; l++) {
            const Impl::Layer &L = I.layers[l];
            LayerPtrs lp{};
            lp.qkvQs = L.qkv.qs; lp.qkvSc = L.qkv.scales; lp.woQs = L.wo.qs; lp.woSc = L.wo.scales;
            lp.w13Qs = L.w13.qs; lp.w13Sc = L.w13.scales; lp.w2Qs = L.w2.qs; lp.w2Sc = L.w2.scales;
            lp.norm0 = L.norm0; lp.norm1 = L.norm1; lp.qNorm = L.qNorm; lp.kNorm = L.kNorm; lp.moeGate = L.moeGate;
            lp.kCache = L.kCache; lp.vCache = L.vCache; lp.kScale = L.kScale; lp.vScale = L.vScale;
            engCheck(dl_engine_set_layer(I.engine, l, &lp), "dl_engine_set_layer");
        }
        engCheck(dl_engine_set_globals(I.engine, &g), "dl_engine_set_globals");
        if (N > 1) {
            // symmetric peer-memory arena, laid out by the engine
            const uint64_t bytes = dl_engine_arena_bytes(I.engine);
            I.vmm = dl_vmm_create(rank_, N, bytes, commTag.c_str(), 1);
            if (!I.vmm) throw std::runtime_error("cannot create the peer-memory arena (CUDA VMM with POSIX file-descriptor handles is required)");
            if (hostBarrier) hostBarrier();      // every rank has bound its bootstrap socket
            engCheck(dl_vmm_connect(I.vmm), "dl_vmm_connect");
            cudaCheck(cudaMemsetAsync(dl_vmm_ptr(I.vmm, rank_), 0, bytes, I.stream), "cudaMemset(arena)");
            cudaCheck(cudaStreamSynchronize(I.stream), "cudaMemset(arena)");
            engCheck(dl_vmm_barrier(I.vmm, 3), "dl_vmm_barrier");   // nobody pushes into an arena that is still being cleared
            CommPtrs cp{};
            cp.nRanks = N; cp.rank = rank_;
            for (uint32_t r = 0; r < N; r++) cp.arena[r] = dl_vmm_ptr(I.vmm, r);
            cp.mcArena = dl_vmm_mc_ptr(I.vmm);
            multicast_ = cp.mcArena != nullptr;
            engCheck(dl_engine_set_comm(I.engine, &cp), "dl_engine_set_comm");
        }
        if (!moe) {
            engCheck(dl_engine_enable_mega(I.engine, 1), "dl_engine_enable_mega");   // falls back per call if the shape is unsupported
            mega_ = true;
        }
        cudaCheck(cudaDeviceSynchronize(), "weight upload");
    } catch (...) {
        release();
        throw;
    }
}

void NativeEngine::release() {
    if (!impl_) return;
    cudaDeviceSynchronize();
    if (impl_->engine) dl_engine_destroy(impl_->engine);
    if (impl_->vmm) dl_vmm_destroy(impl_->vmm);
    for (void *p : impl_->allocations) cudaFree(p);
    if (impl_->stream) cudaStreamDestroy(impl_->stream);
    delete impl_;
    impl_ = nullptr;
}

NativeEngine::~NativeEngine() { release(); }

// Same device-side fusions as distributed_llama_b200/models/loader.py: q|k|v rows concatenated, w1/w3 rows interleaved,
// NeoX (Qwen3) rotary layout re-ordered to adjacent pairs by the repack kernel, q_norm/k_norm permuted alike.
void NativeEngine::uploadWeights(const uint8_t *file) {
    Impl &I = *impl_;
    const uint32_t hd = h_.headDim, dim = h_.dim, ff = ffL_, vocab = vocabL_;
    const uint32_t qDim = headsL_ * hd, kvDim = kvHeadsL_ * hd;
    const bool neox = h_.ropeType == ROPE_FALCON;
    const uint32_t nExp = std::max(1u, h_.nExperts);
    cudaStream_t st = I.stream;

    uint64_t maxRaw = 0;
    for (const TensorEntry &t : dir_) if (t.type == F_Q40) maxRaw = std::max(maxRaw, t.nBytes);
    void *staging = nullptr;
    cudaCheck(cudaMalloc(&staging, maxRaw + 16), "cudaMalloc(staging)");
    auto q40Alloc = [&](uint64_t rows, uint64_t n) {
        Q40Dev w;
        w.qs = dev(rows * (n / 8) * 4);
        w.scales = dev(rows * (n / 32) * 2);
        return w;
    };
    // rows [slice * rowsLocal, (slice + 1) * rowsLocal) of a file tensor: one contiguous byte range (the reference's row split)
    auto repackRows = [&](const TensorEntry &t, const Q40Dev &dst, uint32_t dstStride, uint32_t dstOff, uint32_t headDim, uint32_t rowsLocal,
                          uint32_t slice) {
        const uint64_t rowBytes = (t.n / 32) * 18, bytes = rowBytes * rowsLocal;
        cudaCheck(cudaMemcpyAsync(staging, file + t.offset + (uint64_t)slice * bytes, bytes, cudaMemcpyHostToDevice, st), "cudaMemcpy(weights)");
        engCheck(dl_repack_q40(staging, rowBytes, 0, rowsLocal, (uint32_t)(t.n / 32), dst.qs, dst.scales, dstStride, dstOff, headDim, st), "dl_repack_q40");
        cudaCheck(cudaStreamSynchronize(st), "repack");   // the staging buffer is re-used by the next tensor
        bytesUploaded_ += bytes;
    };
    // columns [slice * colsLocal, (slice + 1) * colsLocal) of every row (the reference's column split, src/nn/nn-core.cpp:307-322):
    // the rank's 18-byte blocks are gathered on the host so that only its bytes cross PCIe
    std::vector<uint8_t> gather;
    auto repackCols = [&](const TensorEntry &t, const Q40Dev &dst, uint32_t dstOff, uint32_t colsLocal, uint32_t slice) {
        const uint64_t rowBytes = (t.n / 32) * 18, locBytes = (uint64_t)(colsLocal / 32) * 18;
        const uint8_t *src = file + t.offset;
        if (locBytes != rowBytes) {
            gather.resize((size_t)t.d * locBytes);
            for (uint64_t r = 0; r < t.d; r++) std::memcpy(gather.data() + r * locBytes, file + t.offset + r * rowBytes + (uint64_t)slice * locBytes, locBytes);
            src = gather.data();
        }
        cudaCheck(cudaMemcpyAsync(staging, src, (size_t)t.d * locBytes, cudaMemcpyHostToDevice, st), "cudaMemcpy(weights)");
        engCheck(dl_repack_q40(staging, locBytes, 0, (uint32_t)t.d, colsLocal / 32, dst.qs, dst.scales, 1, dstOff, 0, st), "dl_repack_q40");
        cudaCheck(cudaStreamSynchronize(st), "repack");
        bytesUploaded_ += (uint64_t)t.d * locBytes;
    };
    auto f32Tensor = [&](const TensorEntry &t, const std::vector<uint32_t> *perm = nullptr) {
        const size_t count = (size_t)t.d * t.n;
        float *p = (float *)dev(count * 4);
        if (perm) {
            std::vector<float> tmp(count);
            const float *src = (const float *)(file + t.offset);
            for (size_t i = 0; i < count; i++) tmp[i] = src[(*perm)[i]];
            cudaCheck(cudaMemcpyAsync(p, tmp.data(), count * 4, cudaMemcpyHostToDevice, st), "cudaMemcpy(f32)");
            cudaCheck(cudaStreamSynchronize(st), "cudaMemcpy(f32)");
        } else {
            cudaCheck(cudaMemcpyAsync(p, file + t.offset, count * 4, cudaMemcpyHostToDevice, st), "cudaMemcpy(f32)");
        }
        bytesUploaded_ += count * 4;
        return p;
    };
    std::vector<uint32_t> perm(hd);   // new[2j] = old[j], new[2j+1] = old[j + hd/2]
    for (uint32_t j = 0; j < hd / 2; j++) { perm[2 * j] = j; perm[2 * j + 1] = j + hd / 2; }

    I.embedding = f32Tensor(I.entry("embedding"));
    I.finalNorm = f32Tensor(I.entry("final_norm"));
    I.wcls = q40Alloc(vocab, dim);
    repackRows(I.entry("final_matmul_logits"), I.wcls, 1, 0, 0, vocab, rank_);
    {
        std::vector<float> table((size_t)seqLen_ * hd);
        buildRopeTable(h_, seqLen_, table.data());
        I.rope = (float *)dev(table.size() * 4);
        cudaCheck(cudaMemcpyAsync(I.rope, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st), "cudaMemcpy(rope)");
        cudaCheck(cudaStreamSynchronize(st), "cudaMemcpy(rope)");
    }
    I.layers.resize(h_.nLayers);
    for (uint32_t l = 0; l < h_.nLayers; l++) {
        Impl::Layer &L = I.layers[l];
        L.qkv = q40Alloc(qkvDim_, dim);
        repackRows(I.entry("block_matmul_q", l), L.qkv, 1, 0, neox ? hd : 0, qDim, rank_);
        repackRows(I.entry("block_matmul_k", l), L.qkv, 1, qDim, neox ? hd : 0, kvDim, kvRank_);
        repackRows(I.entry("block_matmul_v", l), L.qkv, 1, qDim + kvDim, 0, kvDim, kvRank_);
        L.wo = q40Alloc(dim, qDim);
        repackCols(I.entry("block_matmul_wo", l), L.wo, 0, qDim, rank_);
        L.w13 = q40Alloc((uint64_t)nExp * 2 * ff, dim);
        L.w2 = q40Alloc((uint64_t)nExp * dim, ff);
        for (uint32_t e = 0; e < nExp; e++) {
            repackRows(I.entry("block_matmul_w1", l, e), L.w13, 2, e * 2 * ff, 0, ff, rank_);
            repackRows(I.entry("block_matmul_w3", l, e), L.w13, 2, e * 2 * ff + 1, 0, ff, rank_);
            repackCols(I.entry("block_matmul_w2", l, e), L.w2, e * dim, ff, rank_);
        }
        L.norm0 = f32Tensor(I.entry("block_norm_0", l));
        L.norm1 = f32Tensor(I.entry("block_norm_1", l));
        if (h_.qkNorm()) {
            L.qNorm = f32Tensor(I.entry("block_norm_q", l), neox ? &perm : nullptr);
            L.kNorm = f32Tensor(I.entry("block_norm_k", l), neox ? &perm : nullptr);
        }
        if (h_.nExperts > 0) L.moeGate = f32Tensor(I.entry("block_moe_gate", l));
        const size_t kvValues = (size_t)kvHeadsL_ * seqLen_ * hd;
        L.kCache = dev(kvValues * (kvType_ ? 1 : 2));
        L.vCache = dev(kvValues * (kvType_ ? 1 : 2));
        if (kvType_) {   // q80 scale planes, 16 bytes of tail padding for the persistent kernel's aligned bulk copies
            L.kScale = dev(kvValues / 16 + 16);
            L.vScale = dev(kvValues / 16 + 16);
        }
    }
    cudaCheck(cudaStreamSynchronize(st), "weight upload");
    cudaFree(staging);
}

void NativeEngine::setInputs(const int32_t *tokens, uint32_t n, uint32_t pos) {
    std::vector<int32_t> p(n);
    for (uint32_t i = 0; i < n; i++) p[i] = (int32_t)(pos + i);
    Impl &I = *impl_;
    // pageable sources: the copies are staged before the call returns, so the vectors may die right away
    cudaCheck(cudaMemcpyAsync(I.tokens, tokens, n * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(tokens)");
    cudaCheck(cudaMemcpyAsync(I.pos, p.data(), n * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(pos)");
}

void NativeEngine::forward(uint32_t n, int logitsMode, bool greedyAdvance) {
    engCheck(dl_engine_forward(impl_->engine, (int)n, logitsMode, greedyAdvance ? 1 : 0, impl_->stream), "dl_engine_forward");
}

void NativeEngine::prefill(const std::vector<int32_t> &tokens, uint32_t pos) {
    if (pos + tokens.size() > seqLen_) throw std::runtime_error("position beyond the context length");
    engCheck(dl_engine_prefill(impl_->engine, tokens.data(), (uint32_t)tokens.size(), pos, -1, 0, impl_->stream), "dl_engine_prefill");
}

const float *NativeEngine::step(int32_t token, uint32_t pos) {
    if (nRanks_ > 1) throw std::runtime_error("host-side logits are not gathered under tensor parallelism: use stepGreedy / stepSampled");
    if (pos >= seqLen_) throw std::runtime_error("position beyond the context length");
    setInputs(&token, 1, pos);
    forward(1, 1, false);
    Impl &I = *impl_;
    cudaCheck(cudaMemcpyAsync(I.hostLogits.data(), I.logits, (size_t)h_.vocabSize * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(logits)");
    cudaCheck(cudaStreamSynchronize(I.stream), "step");
    return I.hostLogits.data();
}

std::vector<int32_t> NativeEngine::decodeGreedy(int32_t firstToken, uint32_t pos, uint32_t nSteps) {
    if (pos + nSteps > seqLen_) throw std::runtime_error("decode would run past the context length");
    Impl &I = *impl_;
    setInputs(&firstToken, 1, pos);
    engCheck(dl_engine_decode_graph(I.engine, (int)nSteps, I.stream), "dl_engine_decode_graph");
    std::vector<int32_t> out(nSteps);
    cudaCheck(cudaMemcpyAsync(out.data(), I.history + pos + 1, (size_t)nSteps * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(history)");
    cudaCheck(cudaStreamSynchronize(I.stream), "decode");
    return out;
}

std::vector<int32_t> NativeEngine::specRound(NativeEngine &draft, int32_t token, uint32_t pos, uint32_t k, SpecStats &stats) {
    constexpr uint32_t kWords = 12, kHead = 4;
    if (dl_spec_result_words() != kWords) throw std::runtime_error("speculative result block size differs from the library's");
    draft.synchronize();   // the draft's prefills ran on its own stream; the round runs on this engine's
    int32_t out[kWords];
    engCheck(dl_spec_round(impl_->engine, draft.impl_->engine, token, (int)pos, (int)k, 1, out, impl_->stream), "dl_spec_round");
    const uint32_t n = (uint32_t)out[1];
    stats.rounds++;
    stats.drafted += (uint32_t)out[2];
    stats.accepted += (uint32_t)out[0];
    stats.emitted += n;
    return std::vector<int32_t>(out + kHead, out + kHead + n);
}

int32_t NativeEngine::stepGreedy(int32_t token, uint32_t pos) {
    if (pos >= seqLen_) throw std::runtime_error("position beyond the context length");
    Impl &I = *impl_;
    setInputs(&token, 1, pos);
    engCheck(dl_engine_decode_graph(I.engine, 1, I.stream), "dl_engine_decode_graph");
    if (lpK_ >= 0) logprobsAfterDraw(1, 1u, 0, 0);
    int32_t next = 0;   // the arg-max kernel leaves the sampled token in tokens[0] (and advances pos[0]) on the device
    cudaCheck(cudaMemcpyAsync(&next, I.tokens, 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(token)");
    cudaCheck(cudaStreamSynchronize(I.stream), "stepGreedy");
    if (nRanks_ > 1 && dl_engine_aborted(I.engine)) throw std::runtime_error("device-side wait timed out: a tensor-parallel peer stopped responding");
    return next;
}

void NativeEngine::seedSampler(uint64_t seed) { engCheck(dl_engine_sampler_seed(impl_->engine, seed), "dl_engine_sampler_seed"); }

int32_t NativeEngine::stepSampled(int32_t token, uint32_t pos, float temperature, float topp) {
    if (pos >= seqLen_) throw std::runtime_error("position beyond the context length");
    Impl &I = *impl_;
    setInputs(&token, 1, pos);
    forward(1, 1, false);
    engCheck(dl_engine_sample(I.engine, temperature, topp, I.stream), "dl_engine_sample");
    if (lpK_ >= 0) logprobsAfterDraw(1, 1u, 0, kLogprobsControlled);
    int32_t next = 0;   // the sampler leaves the drawn token in tokens[0]
    cudaCheck(cudaMemcpyAsync(&next, I.tokens, 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(token)");
    cudaCheck(cudaStreamSynchronize(I.stream), "stepSampled");
    if (dl_engine_aborted(I.engine)) throw std::runtime_error("device-side wait timed out: a tensor-parallel peer stopped responding");
    return next;
}

uint64_t NativeEngine::samplerState() { return (uint64_t)dl_engine_sampler_state(impl_->engine); }

void NativeEngine::setSamplingControls(float presence, float frequency, const std::vector<std::pair<int32_t, float>> &bias, uint32_t rowMask) {
    std::vector<int32_t> ids;
    std::vector<float> vals;
    for (const auto &b : bias) { ids.push_back(b.first); vals.push_back(b.second); }
    engCheck(dl_engine_set_sampling_controls(impl_->engine, presence, frequency, ids.data(), vals.data(), (int)ids.size(), rowMask,
                                             impl_->stream),
             "dl_engine_set_sampling_controls");
}

void NativeEngine::setSamplingFilters(uint32_t topK, float minP) {
    engCheck(dl_engine_set_sampling_filters(impl_->engine, topK, minP), "dl_engine_set_sampling_filters");
}

void NativeEngine::seedChoiceSamplers(const std::vector<uint64_t> &seeds) {
    std::vector<unsigned long long> s(seeds.begin(), seeds.end());
    engCheck(dl_engine_sampler_seed_rows(impl_->engine, s.data(), (int)s.size()), "dl_engine_sampler_seed_rows");
}

static uint32_t choiceBatch(uint32_t n) { uint32_t nb = 1; while (nb < n) nb *= 2; return nb; }

std::vector<int32_t> NativeEngine::choicesFirst(int32_t token, uint32_t P, uint32_t n, float temperature, float topp) {
    if (!supportsChoices(n) || P >= seqLen_) throw std::runtime_error("choices: unsupported batch or position");
    Impl &I = *impl_;
    setInputs(&token, 1, P);
    forward(1, 1, false);
    const uint32_t nb = choiceBatch(n), mask = ((1u << nb) - 1u) & ~((1u << n) - 1u);
    engCheck(dl_engine_sample_rows(I.engine, (int)nb, mask, temperature, topp, 1, I.stream), "dl_engine_sample_rows");
    if (lpK_ >= 0) logprobsAfterDraw(n, (1u << n) - 1u, 1, kLogprobsControlled | kLogprobsSharedRow);
    std::vector<int32_t> out(n);
    cudaCheck(cudaMemcpyAsync(out.data(), I.tokens, n * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(tokens)");
    cudaCheck(cudaStreamSynchronize(I.stream), "choicesFirst");
    if (dl_engine_aborted(I.engine)) throw std::runtime_error("device-side wait timed out: a tensor-parallel peer stopped responding");
    return out;
}

std::vector<int32_t> NativeEngine::choicesStep(const std::vector<int32_t> &tokens, uint32_t P, uint32_t C, uint32_t j, uint32_t activeMask,
                                               float temperature, float topp) {
    const uint32_t n = (uint32_t)tokens.size(), nb = choiceBatch(n);
    if (!supportsChoices(n) || C < 1 || j >= C || (uint64_t)P + 1 + (uint64_t)n * C > seqLen_) throw std::runtime_error("choices: rows beyond the context");
    Impl &I = *impl_;
    std::vector<int32_t> t(tokens), p(nb, (int32_t)(P + 1 + j));
    t.resize(nb, 0);
    const uint32_t mask = ~activeMask & ((1u << nb) - 1u);
    cudaCheck(cudaMemcpyAsync(I.tokens, t.data(), nb * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(tokens)");
    cudaCheck(cudaMemcpyAsync(I.pos, p.data(), nb * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(pos)");
    engCheck(dl_engine_choices_forward(I.engine, (int)nb, P, C, j, mask, I.stream), "dl_engine_choices_forward");
    engCheck(dl_engine_sample_rows(I.engine, (int)nb, mask, temperature, topp, 0, I.stream), "dl_engine_sample_rows");
    if (lpK_ >= 0) logprobsAfterDraw(n, activeMask & ((1u << n) - 1u), 1, kLogprobsControlled);
    std::vector<int32_t> out(n);
    cudaCheck(cudaMemcpyAsync(out.data(), I.tokens, n * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(tokens)");
    cudaCheck(cudaStreamSynchronize(I.stream), "choicesStep");
    if (dl_engine_aborted(I.engine)) throw std::runtime_error("device-side wait timed out: a tensor-parallel peer stopped responding");
    return out;
}

void NativeEngine::setSlots(uint32_t n, bool paged) {
    engCheck(dl_engine_set_slot_cache(impl_->engine, paged ? 1 : 0), "dl_engine_set_slot_cache");
    engCheck(dl_engine_set_slots(impl_->engine, n), "dl_engine_set_slots");
    slots_ = n;
}

bool NativeEngine::slotReserve(uint32_t slot, uint32_t rows) {
    const int rc = dl_engine_slot_reserve(impl_->engine, slot, rows);
    if (rc == dl::kEngineErrPoolShort) return false;
    engCheck(rc, "dl_engine_slot_reserve");
    return true;
}

void NativeEngine::slotTrim(uint32_t slot, uint32_t rows) { engCheck(dl_engine_slot_trim(impl_->engine, slot, rows), "dl_engine_slot_trim"); }
void NativeEngine::slotRelease(uint32_t slot) { engCheck(dl_engine_slot_release(impl_->engine, slot), "dl_engine_slot_release"); }
uint32_t NativeEngine::freePages() const { return dl_engine_free_pages(impl_->engine); }
uint32_t NativeEngine::slotPageCount(uint32_t slot) const {
    const int n = dl_engine_slot_pages(impl_->engine, slot, nullptr, 0);
    return n > 0 ? (uint32_t)n : 0u;
}

uint32_t NativeEngine::slotLen() const { return dl_engine_slot_len(impl_->engine); }

void NativeEngine::slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) {
    if (pos + tokens.size() > slotLen()) throw std::runtime_error("position beyond the slot length");
    engCheck(dl_engine_prefill(impl_->engine, tokens.data(), (uint32_t)tokens.size(), pos, (int)slot, 0, impl_->stream), "dl_engine_prefill");
}

void NativeEngine::slotCopy(uint32_t src, uint32_t dst, uint32_t P) {
    engCheck(dl_engine_slot_copy(impl_->engine, src, dst, P, impl_->stream), "dl_engine_slot_copy");
}

void NativeEngine::slotSampling(uint32_t slot, uint64_t seed, float temperature, float topp, float presence, float frequency,
                                const std::vector<std::pair<int32_t, float>> &bias) {
    std::vector<int32_t> ids;
    std::vector<float> vals;
    for (const auto &b : bias) { ids.push_back(b.first); vals.push_back(b.second); }
    engCheck(dl_engine_slot_sampling(impl_->engine, slot, seed, temperature, topp, presence, frequency, ids.data(), vals.data(), (int)ids.size(),
                                     impl_->stream), "dl_engine_slot_sampling");
}

void NativeEngine::slotFilters(uint32_t slot, uint32_t topK, float minP) {
    engCheck(dl_engine_slot_filters(impl_->engine, slot, topK, minP), "dl_engine_slot_filters");
}

std::vector<int32_t> NativeEngine::slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask) {
    if (tokens.size() != slots_ || pos.size() != slots_) throw std::runtime_error("slotsStep: one token and position per slot");
    std::vector<int32_t> out(slots_, -1);
    const uint32_t inactive = ~activeMask & ((1u << slots_) - 1u);
    engCheck(dl_engine_slots_step(impl_->engine, tokens.data(), pos.data(), inactive, out.data(), impl_->stream), "dl_engine_slots_step");
    return out;
}

static constexpr size_t kLogprobsRows = 8;   // the widest draw: one row per choice or slot

void NativeEngine::logprobsAfterDraw(uint32_t rows, uint32_t rowMask, int firstRow, int flags) {
    if (nRanks_ > 1) throw std::runtime_error("logprobs are not supported under tensor parallelism yet");
    Impl &I = *impl_;
    if (!lpDev_) lpDev_ = (int32_t *)dev(kLogprobsRows * kApiLogprobsWords * sizeof(int32_t));
    const std::vector<int32_t> k(rows, lpK_);
    engCheck(dl_engine_logprobs(I.engine, (int)rows, rowMask, k.data(), firstRow, flags, lpDev_, I.stream), "dl_engine_logprobs");
    lpHost_.assign((size_t)rows * kApiLogprobsWords, 0);
    cudaCheck(cudaMemcpyAsync(lpHost_.data(), lpDev_, lpHost_.size() * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(logprobs)");
}

void NativeEngine::logprobsHostDraw(int32_t token, uint32_t n, const std::vector<float> &bias, const std::vector<uint32_t> &counts, float presence,
                                    float frequency) {
    if (nRanks_ > 1) throw std::runtime_error("logprobs are not supported under tensor parallelism yet");
    Impl &I = *impl_;
    if (!lpDev_) lpDev_ = (int32_t *)dev(kLogprobsRows * kApiLogprobsWords * sizeof(int32_t));
    // scratch: chosen id, then the bias and counts rows of the host sampler (uploaded only when it has controls)
    const size_t V = h_.vocabSize;
    if (!lpScratch_) lpScratch_ = (uint8_t *)dev(16 + 8 * V);
    int32_t *chosen = (int32_t *)lpScratch_;
    float *biasDev = bias.empty() ? nullptr : (float *)(lpScratch_ + 16);
    uint32_t *countsDev = counts.empty() ? nullptr : (uint32_t *)(lpScratch_ + 16 + 4 * V);
    cudaCheck(cudaMemcpyAsync(chosen, &token, 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(logprobs)");
    if (biasDev) cudaCheck(cudaMemcpyAsync(biasDev, bias.data(), std::min(bias.size(), V) * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(bias)");
    if (countsDev) cudaCheck(cudaMemcpyAsync(countsDev, counts.data(), std::min(counts.size(), V) * 4, cudaMemcpyHostToDevice, I.stream), "cudaMemcpy(counts)");
    const int k = lpK_;
    engCheck(dl_logprobs_rows(I.logits, 0, std::min<uint32_t>(n, h_.vocabSize), 1, 1u, &k, chosen, biasDev, 0, countsDev, 0, presence, frequency,
                              nullptr, lpDev_, I.stream), "dl_logprobs_rows");
    lpHost_.assign(kApiLogprobsWords, 0);
    cudaCheck(cudaMemcpyAsync(lpHost_.data(), lpDev_, lpHost_.size() * 4, cudaMemcpyDeviceToHost, I.stream), "cudaMemcpy(logprobs)");
    cudaCheck(cudaStreamSynchronize(I.stream), "logprobs");   // the host vectors are read by the copies above
}

void NativeEngine::slotLogprobs(uint32_t slot, int k) { engCheck(dl_engine_slot_logprobs(impl_->engine, slot, k), "dl_engine_slot_logprobs"); }

std::vector<int32_t> NativeEngine::slotsStepLogprobs(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t activeMask,
                                                     std::vector<int32_t> &blocks) {
    if (tokens.size() != slots_ || pos.size() != slots_) throw std::runtime_error("slotsStep: one token and position per slot");
    std::vector<int32_t> out(slots_, -1);
    blocks.assign((size_t)slots_ * kApiLogprobsWords, 0);
    for (uint32_t b = 0; b < slots_; b++) blocks[(size_t)b * kApiLogprobsWords + 2] = -1;   // rows the step leaves alone keep k = -1
    const uint32_t inactive = ~activeMask & ((1u << slots_) - 1u);
    engCheck(dl_engine_slots_step_logprobs(impl_->engine, tokens.data(), pos.data(), inactive, out.data(), blocks.data(), impl_->stream),
             "dl_engine_slots_step_logprobs");
    return out;
}

uint64_t NativeEngine::syncNs() const { return nRanks_ > 1 ? (uint64_t)dl_engine_sync_ns(impl_->engine) : 0; }

void NativeEngine::linkBytes(uint32_t nTokens, uint64_t &sent, uint64_t &received) const {
    sent = received = 0;
    if (nRanks_ <= 1) return;
    const uint64_t perAr = (uint64_t)nTokens * h_.dim * 8;
    sent = 2ull * h_.nLayers * perAr * (multicast_ ? 1 : nRanks_ - 1);
    received = 2ull * h_.nLayers * perAr * (nRanks_ - 1);
}

void NativeEngine::synchronize() { cudaCheck(cudaStreamSynchronize(impl_->stream), "synchronize"); }

void NativeEngine::setVocabLimit(uint32_t limit) {
    if (limit >= h_.vocabSize) limit = 0;
    engCheck(dl_engine_set_vocab_limit(impl_->engine, limit), "dl_engine_set_vocab_limit");
}

}  // namespace dl
