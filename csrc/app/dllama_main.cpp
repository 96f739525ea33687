// `dllama-native {inference|perplexity|chat}` — the reference CLI (src/dllama.cpp:13-285, flag table src/app.cpp:24-135)
// as one native binary: C++ tokenizer / sampler / chat templates (csrc/host), native engine driver (native_engine.cpp), CUDA
// kernels from _cuda.so. No interpreter in the process.
//
// `--gpus N` (tensor parallel over the GPUs of one NVSwitch box) is the reference's root + `dllama worker` processes
// (src/dllama.cpp:260-285, src/app.cpp:306-365) without sockets: the root forks one worker process per extra GPU *before* CUDA is
// initialised; every process loads its slice of the model, joins the peer-memory arena (CUDA VMM handles passed over unix sockets,
// csrc/cuda/comm_vmm.cu) and the workers then mirror the root's engine calls, which reach them through a control block in an
// anonymous shared mapping (the reference's LlmControlPacket, src/app.hpp:46-49). A worker that dies is noticed by the root
// (waitpid) and the root's death by the workers (getppid): nobody waits forever. The all-reduces themselves run inside the
// kernels over NVLink.
#include <sys/mman.h>
#include <sys/prctl.h>
#include <sys/wait.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <iostream>
#include <memory>
#include <new>
#include <csignal>
#include <stdexcept>
#include <string>
#include <vector>

#include "../host/text.hpp"
#include "api_server.hpp"
#include "native_engine.hpp"
#include "tp_job.hpp"

using namespace dl;

namespace {

struct Args {
    std::string mode, model, tokenizer, prompt, chatTemplate, bufferFloatType = "q80";
    bool hasPrompt = false, help = false;
    uint32_t steps = 0, maxSeqLen = 0;
    uint32_t kvType = 0;    // --kv-cache-float-type: 0 = bf16, 1 = q80
    float temperature = 0.8f, topp = 0.9f;
    float presencePenalty = 0.f, frequencyPenalty = 0.f;
    uint32_t topK = 0;      // sampling filters (Sampler::setFilters), 0 = off
    float minP = 0.f;
    uint64_t seed = (uint64_t)std::time(nullptr);
    int gpuIndex = 0;
    uint32_t gpus = 1, workers = 0;
    std::string draftModel;   // --draft-model: greedy speculative decoding with this smaller model (one GPU)
    uint32_t draftTokens = 3;
};

const char *kUsage =
    "Usage: dllama-native {inference|perplexity|chat} --model <path> --tokenizer <path>\n"
    "        [--prompt <text>] [--steps <n>] [--temperature <t>] [--topp <p>] [--presence-penalty <p>] [--frequency-penalty <f>]\n"
    "        [--top-k <k>] [--min-p <p>]   sampling filters of sampled draws (default 0 = off)\n"
    "        [--seed <s>] [--max-seq-len <n>] [--kv-cache-float-type {bf16|q80}]\n"
    "        [--chat-template {llama2|llama3|deepSeek3|chatml}] [--buffer-float-type q80] [--gpu-index <i>]\n"
    "        [--gpus <n>]   tensor parallel over GPUs gpu-index .. gpu-index + n - 1 of this machine (one process per GPU)\n"
    "        [--draft-model <path>] [--draft-tokens {1|3|7}]  greedy speculative decoding: the draft proposes k tokens a round (default 3)\n"
    "        (accepted for drop-in compatibility and ignored: --nthreads --net-turbo --gpu-segments --workers --host --port)\n";

Args parse(int argc, char **argv) {
    Args a;
    int i = 1;
    if (i < argc && argv[i][0] != '-') a.mode = argv[i++];
    while (i < argc) {
        const std::string name = argv[i];
        if (name == "--help" || name == "-h" || name == "--usage") { a.help = true; return a; }
        if (name == "--workers") {   // variadic until the next flag
            i++;
            while (i < argc && argv[i][0] != '-') { i++; a.workers++; }
            continue;
        }
        if (i + 1 >= argc) throw std::runtime_error("Missing value for " + name);
        const std::string value = argv[i + 1];
        if (name == "--model") a.model = value;
        else if (name == "--tokenizer") a.tokenizer = value;
        else if (name == "--prompt") { a.prompt = value; a.hasPrompt = true; }
        else if (name == "--steps") a.steps = (uint32_t)std::stoul(value);
        else if (name == "--temperature") a.temperature = std::stof(value);
        else if (name == "--topp") a.topp = std::stof(value);
        else if (name == "--presence-penalty") a.presencePenalty = parsePenalty(name, value);
        else if (name == "--frequency-penalty") a.frequencyPenalty = parsePenalty(name, value);
        else if (name == "--top-k") a.topK = parseTopK(name, value);
        else if (name == "--min-p") a.minP = parseMinP(name, value);
        else if (name == "--seed") a.seed = std::stoull(value);
        else if (name == "--max-seq-len") a.maxSeqLen = (uint32_t)std::stoul(value);
        else if (name == "--kv-cache-float-type") a.kvType = parseKvCacheFloatType(value);
        else if (name == "--chat-template") a.chatTemplate = value;
        else if (name == "--buffer-float-type") a.bufferFloatType = value;
        else if (name == "--gpu-index") a.gpuIndex = std::max(0, std::stoi(value));
        else if (name == "--gpus") a.gpus = (uint32_t)std::max(1, std::stoi(value));
        else if (name == "--draft-model") a.draftModel = value;
        else if (name == "--draft-tokens") a.draftTokens = (uint32_t)std::max(0, std::stoi(value));
        else if (name == "--nthreads" || name == "--net-turbo" || name == "--gpu-segments" || name == "--host" || name == "--port") {}
        else throw std::runtime_error("Unknown option: " + name);
        i += 2;
    }
    return a;
}

double nowMs() {
    using namespace std::chrono;
    return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

struct App {
    Args args;
    TpJob &job;
    NativeEngine engine;
    Tokenizer tokenizer;
    Sampler sampler;
    TpEngine tp;
    std::unique_ptr<NativeEngine> draft;   // --draft-model: the target's context length and KV-cache storage
    SpecStats specStats;
    App(const Args &a, TpJob &j)
        : args(a), job(j), engine(a.model, a.maxSeqLen, a.gpuIndex + (int)j.rank, j.rank, j.nRanks, j.tag, [&j] { j.barrier(); }, a.kvType),
          tokenizer(a.tokenizer),
          sampler(std::min<uint32_t>(tokenizer.vocabSize(), engine.header().vocabSize), a.temperature, a.topp, a.seed), tp{engine, j} {
        // sampling ranges over the tokenizer's vocabulary (reference src/app.cpp:243-246); padded embedding rows never win
        engine.setVocabLimit(tokenizer.vocabSize());
        sampler.setControls(a.presencePenalty, a.frequencyPenalty, {});
        sampler.setFilters(a.topK, a.minP);
        if (!a.draftModel.empty()) {
            const ModelHeader dh = loadModelHeader(a.draftModel, engine.seqLen());
            const std::string why = draftRefusal(a.draftTokens, j.nRanks, 1, &engine.header(), &dh);
            if (!why.empty()) throw std::runtime_error(why);
            draft.reset(new NativeEngine(a.draftModel, engine.seqLen(), a.gpuIndex, 0, 1, std::string(), std::function<void()>(), a.kvType));
            draft->setVocabLimit(tokenizer.vocabSize());
        }
    }

    void prefill(const std::vector<int32_t> &tokens, uint32_t pos) {
        tp.prefill(tokens, pos);
        if (draft && !tokens.empty()) draft->prefill(tokens, pos);
    }

    int32_t next(int32_t token, uint32_t pos) { return tp.next(token, pos, sampler); }

    // the tokens of one step: a speculative round for plain greedy decoding with a draft, else one token
    std::vector<int32_t> nextTokens(int32_t token, uint32_t pos) {
        if (draft && sampler.temperature() == 0.f && !sampler.controlsActive())
            return engine.specRound(*draft, token, pos, args.draftTokens, specStats);
        return {next(token, pos)};
    }
};

void inference(App &app) {
    const Args &a = app.args;
    if (!a.hasPrompt) throw std::runtime_error("Prompt is required");
    if (a.steps == 0) throw std::runtime_error("Number of steps is required");
    const ModelHeader &h = app.engine.header();
    const std::vector<int32_t> tokens = app.tokenizer.encode(a.prompt, true, true);
    const uint32_t nIn = (uint32_t)tokens.size();
    if (nIn > h.seqLen) throw std::runtime_error("The number of prompt tokens is greater than the sequence length");
    if (nIn > a.steps) throw std::runtime_error("The number of prompt tokens is greater than the number of steps");
    std::printf("%s\n", a.prompt.c_str());
    double evalMs = 0, predMs = 0, syncMs = 0;
    uint32_t pos = 0;
    const uint32_t chunk = 192;   // tokens per tensor-core prefill launch (the reference feeds 32 per forward)
    while (pos + 1 < nIn) {
        const uint32_t n = std::min(chunk, nIn - 1 - pos);
        const double t0 = nowMs();
        app.prefill(std::vector<int32_t>(tokens.begin() + pos, tokens.begin() + pos + n), pos);
        app.engine.synchronize();
        const double dt = nowMs() - t0;
        evalMs += dt;
        uint64_t sent = 0, recv = 0;
        app.engine.linkBytes(n, sent, recv);
        std::printf("🔷️ Eval%5d ms Sync%5d ms | Sent%6d kB Recv%6d kB | (%u tokens)\n", (int)dt, 0, (int)(sent / 1024), (int)(recv / 1024), n);
        pos += n;
    }
    std::fflush(stdout);
    int32_t token = tokens[pos];
    app.tokenizer.resetDecoder();
    app.sampler.beginCompletion();
    const uint32_t maxPos = std::min(h.seqLen, a.steps);
    uint32_t nPred = 0;
    while (pos < maxPos) {
        const double t0 = nowMs();
        const uint64_t sync0 = app.engine.syncNs();
        // a speculative round emits several tokens: each line shows its share of the round's time
        const std::vector<int32_t> toks = app.nextTokens(token, pos);
        const double dt = nowMs() - t0;
        predMs += dt;
        syncMs += (double)(app.engine.syncNs() - sync0) * 1e-6;
        for (const int32_t t : toks) {
            token = t;
            uint64_t sent = 0, recv = 0;
            app.engine.linkBytes(1, sent, recv);
            const std::string piece = app.tokenizer.decode(token);
            std::printf("🔶 Pred%5d ms Sync%5d ms | Sent%6d kB Recv%6d kB | %s\n", (int)(dt / (double)toks.size()),
                        (int)((double)(app.engine.syncNs() - sync0) * 1e-6), (int)(sent / 1024), (int)(recv / 1024),
                        piece.empty() ? "~" : piece.c_str());
            std::fflush(stdout);
            pos++;
            nPred++;
            if (pos >= maxPos) break;
        }
    }
    const uint32_t nEval = nIn - 1;
    std::printf("\nEvaluation\n   nBatches: %u\n    nTokens: %u\n", chunk, nEval);
    if (nEval > 0 && evalMs > 0) std::printf("   tokens/s: %3.2f (%3.2f ms/tok)\n", nEval * 1000.0 / evalMs, evalMs / nEval);
    std::printf("Prediction\n    nTokens: %u\n", nPred);
    if (nPred > 0 && predMs > 0) std::printf("   tokens/s: %3.2f (%3.2f ms/tok)\n", nPred * 1000.0 / predMs, predMs / nPred);
    if (app.job.nRanks > 1 && nPred > 0) std::printf("   syncTime: %3.3f ms/tok waiting for peers inside the fused all-reduces\n", syncMs / nPred);
    if (app.draft) std::printf("%s\n", app.specStats.line().c_str());
}

void perplexity(App &app) {
    const Args &a = app.args;
    if (app.job.nRanks > 1) throw std::runtime_error("perplexity needs the full logits on the host: run it on one GPU (or through ./dllama perplexity --gpus N)");
    if (!a.hasPrompt) throw std::runtime_error("Prompt is required");
    const ModelHeader &h = app.engine.header();
    const std::vector<int32_t> tokens = app.tokenizer.encode(a.prompt, true, true);
    const size_t n = tokens.size();
    if (n > h.seqLen) throw std::runtime_error("The number of prompt tokens is greater than the sequence length");
    std::printf("Evaluating %zu tokens...\n", n);
    double total = 0;
    std::vector<float> probs(h.vocabSize);
    for (size_t pos = 0; pos + 1 < n; pos++) {
        const float *logits = app.engine.step(tokens[pos], (uint32_t)pos);
        std::memcpy(probs.data(), logits, (size_t)h.vocabSize * sizeof(float));
        softmaxInPlace(probs.data(), h.vocabSize);
        const double p = probs[tokens[pos + 1]];
        total += std::log(std::max(p, 1e-30));
        std::printf("%5zu / %zu, prob=%f\n", pos + 1, n - 1, p);
    }
    const double avg = total / (double)std::max<size_t>(1, n - 1);
    std::printf("\nResults\n   perplexity: %f (lower = better)\n   avgLogProb: %f\n   bitPerToken: %f\n", std::exp(-avg), avg, -avg / std::log(2.0));
}

bool readLine(const char *prompt, std::string &out) {
    std::printf("%s", prompt);
    std::fflush(stdout);
    return (bool)std::getline(std::cin, out);
}

void chat(App &app) {
    const ModelHeader &h = app.engine.header();
    const TokenizerData &td = app.tokenizer.data();
    std::vector<std::string> stops;
    for (int32_t id : td.eosIds) stops.push_back(td.vocab[(size_t)id]);
    size_t maxStop = 0;
    for (const std::string &s : stops) maxStop = std::max(maxStop, s.size());
    const ChatTemplateType type = app.args.chatTemplate.empty() ? TEMPLATE_UNKNOWN : parseChatTemplateType(app.args.chatTemplate);
    ChatTemplateGenerator gen(type, td.chatTemplate, stops.empty() ? std::string() : stops[0]);
    std::printf("⭐ Chat template: %s\n", chatTemplateTypeName(gen.type()));
    for (const std::string &s : stops) std::printf("🛑 Stop: %s\n", s.c_str());
    EosDetector det(td.eosIds, stops, (int)maxStop, (int)maxStop);

    std::string sysPrompt;
    readLine("💻 System prompt (optional): ", sysPrompt);
    std::vector<ChatItem> items;
    if (!sysPrompt.empty()) items.push_back({"system", sysPrompt});
    uint32_t pos = 0;
    while (pos < h.seqLen) {
        std::string user;
        while (user.empty())
            if (!readLine("\n👱 User\n> ", user)) return;
        items.push_back({"user", user});
        const GeneratedChat g = gen.generate(items, true);
        const std::vector<int32_t> tokens = app.tokenizer.encode(g.content, pos == 0, true);
        const uint32_t end = std::min<uint32_t>(h.seqLen, pos + (uint32_t)tokens.size() - 1);
        const uint32_t n = end - pos;
        app.prefill(std::vector<int32_t>(tokens.begin(), tokens.begin() + n), pos);
        pos += n;
        int32_t token = n < tokens.size() ? tokens[n] : tokens.back();
        app.tokenizer.resetDecoder();
        det.reset();
        app.sampler.beginCompletion();
        std::printf("\n🤖 Assistant\n");
        if (!g.publicPrompt.empty()) std::printf("%s", g.publicPrompt.c_str());
        bool eos = false;
        while (pos < h.seqLen && !eos) {
            for (const int32_t t : app.nextTokens(token, pos)) {
                token = t;
                const std::string piece = app.tokenizer.decode(token);
                const EosDetectorResult kind = det.append(token, piece);
                if (kind == NOT_EOS || kind == EOS) {
                    const std::string delta = det.getDelta();
                    if (!delta.empty()) { std::printf("%s", delta.c_str()); std::fflush(stdout); }
                    det.reset();
                }
                pos++;
                eos = kind == EOS;
                if (eos || pos >= h.seqLen) break;
            }
        }
        items.clear();
    }
    std::printf("(end of context)\n");
    if (app.draft) std::printf("%s\n", app.specStats.line().c_str());
}

}  // namespace

int main(int argc, char **argv) {
    try {
        const Args a = parse(argc, argv);
        if (a.help || a.mode.empty()) { std::printf("%s", kUsage); return 0; }
        if (a.mode == "worker")
            throw std::runtime_error("workers are forked by the root: dllama-native <mode> --gpus N");
        if (a.mode != "inference" && a.mode != "perplexity" && a.mode != "chat") throw std::runtime_error("Unsupported mode");
        if (a.model.empty()) throw std::runtime_error("Model is required");
        if (a.tokenizer.empty()) throw std::runtime_error("Tokenizer is required");
        if (a.bufferFloatType != "q80") throw std::runtime_error("This version supports only Q40 weights with Q80 sync type");
        if (!a.draftModel.empty()) {   // refused before any process or GPU work
            const std::string why = draftRefusal(a.draftTokens, a.gpus + a.workers, 1);
            if (!why.empty()) throw std::runtime_error(why);
        }
        // ---- tensor-parallel job: fork the workers before CUDA exists in this process ----
        TpJob job;
        job.create(a.gpus);
        job.reapChildren = true;
        std::vector<pid_t> children;
        if (job.nRanks > 1) {
            const pid_t rootPid = getpid();
            std::fflush(stdout);
            for (uint32_t r = 1; r < job.nRanks; r++) {
                const pid_t pid = fork();
                if (pid < 0) throw std::runtime_error("fork failed");
                if (pid == 0) {
                    prctl(PR_SET_PDEATHSIG, SIGKILL);
                    job.rank = r; job.reapChildren = false; job.parentPid = rootPid;
                    std::fclose(stdin);
                    _exit(tpWorkerMain(a.model, a.tokenizer, a.maxSeqLen, a.gpuIndex, job, a.kvType));
                }
                children.push_back(pid);
            }
        }
        struct Reaper {   // root: tell the workers to leave and collect them, whatever happens
            TpJob &job; std::vector<pid_t> &children;
            ~Reaper() { if (job.nRanks > 1 && job.rank == 0) { job.sendExit(); tpReap(children); } }
        } reaper{job, children};
        std::unique_ptr<App> appPtr;
        try {
            appPtr.reset(new App(a, job));
            if (job.nRanks > 1) job.barrier();   // every rank has its weights
        } catch (const std::exception &e) {
            job.fail(e.what());
            throw;
        }
        App &app = *appPtr;
        const ModelHeader &h = app.engine.header();
        if (app.tokenizer.vocabSize() != h.vocabSize)
            std::printf("Tokenizer vocab size (%u) does not match the model vocab size (%u)\n", app.tokenizer.vocabSize(), h.vocabSize);
        std::printf("%s", app.tokenizer.describe().c_str());
        std::printf("%s", describeModelHeader(h).c_str());
        std::printf("📀 RequiredMemory: %llu MB\n", (unsigned long long)((requiredDeviceBytes(h, job.nRanks, 0) + kvCacheBytes(h, job.nRanks, a.kvType)) / (1024 * 1024)));
        if (job.nRanks > 1)
            std::printf("🔗 %u GPUs (one process each), all-reduce inside the kernels over %s\n", job.nRanks,
                        app.engine.multicast() ? "the NVSwitch multicast mapping (multimem.st)" : "NVLink peer memory");
        std::printf("🧠 GPU %d: sm_90a kernels, %s decode; %.2f GB of weights uploaded%s\n", a.gpuIndex,
                    app.engine.persistentKernel() ? "persistent-kernel" : "multi-kernel", app.engine.bytesUploaded() / 1e9,
                    job.nRanks > 1 ? " by this rank" : "");
        std::printf("💿 Weights loaded\n");
        if (a.mode == "inference") inference(app);
        else if (a.mode == "perplexity") perplexity(app);
        else chat(app);
        return 0;
    } catch (const std::exception &e) {
        std::printf("🚨 Critical error: %s\n", e.what());
        return 1;
    }
}
