// pybind11 surface of the host library (`distributed_llama_b200._host`).
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "model_format.hpp"
#include "quants.hpp"
#include "slot_scheduler.hpp"
#include "text.hpp"

namespace py = pybind11;
using namespace dl;

using F32Array = py::array_t<float, py::array::c_style | py::array::forcecast>;
using U8Array = py::array_t<uint8_t, py::array::c_style | py::array::forcecast>;

static py::bytes asBytes(const std::string &s) { return py::bytes(s.data(), s.size()); }

// SlotScheduler over Python objects (distributed_llama_b200.api.SlotScheduler). run() holds the GIL except while it sleeps, so
// every hook and backend call below runs with it.
namespace {
// A Python int as the engine takes a seed: modulo 2^64.
uint64_t seed64(const py::handle &v) {
    const unsigned long long s = PyLong_AsUnsignedLongLongMask(v.ptr());
    if (PyErr_Occurred()) throw py::error_already_set();
    return s;
}

// A distributed_llama_b200.api.SlotRequest: its fields and hooks.
struct PySlotRequest {
    py::object o;
    uint32_t n() const { return o.attr("n").cast<uint32_t>(); }
    bool greedy() const { return o.attr("temperature").cast<double>() == 0.0; }
    std::optional<uint64_t> seed() const {
        const py::object s = o.attr("seed");
        return s.is_none() ? std::nullopt : std::optional<uint64_t>(seed64(s));
    }
    int64_t maxTokens() const {   // past int64: no limit but the slot's
        int over = 0;
        const long long v = PyLong_AsLongLongAndOverflow(o.attr("max_tokens").ptr(), &over);
        if (PyErr_Occurred()) throw py::error_already_set();
        return over ? (over > 0 ? INT64_MAX : -1) : v;
    }
    int logprobs() const {
        const py::object k = o.attr("logprobs");
        return k.is_none() ? -1 : k.cast<int>();
    }
    size_t cachedPrefix(uint32_t slot) const { return o.attr("cached_prefix")(slot).cast<size_t>(); }
    uint32_t promptLen(uint32_t slot) const { return o.attr("prompt_len")(slot).cast<uint32_t>(); }
    SlotPrompt prepare(uint32_t slot) const {
        const py::tuple t(o.attr("prepare")(slot));
        return {t[0].cast<std::vector<int32_t>>(), t[1].cast<uint32_t>(), t[2].cast<int32_t>(), t[3].cast<uint32_t>()};
    }
    void onLogprobs(uint32_t i, const py::object &entry) const { o.attr("on_logprobs")(i, entry); }
    bool onToken(uint32_t i, int32_t token) const { return py::bool_(o.attr("on_token")(i, token)).cast<bool>(); }
    void finish(const std::vector<std::vector<int32_t>> &out, const std::vector<uint32_t> &slots, uint32_t P) const {
        o.attr("finish")(out, slots, P);
    }
    // A hook's exception goes on as the same object; the scheduler's own refusals as ValueError.
    void fail(std::exception_ptr error, const std::vector<uint32_t> &slots) const {
        py::object e;
        try {
            std::rethrow_exception(error);
        } catch (const py::error_already_set &x) {
            if (!x.matches(PyExc_Exception)) throw;   // KeyboardInterrupt, SystemExit: out of run()
            e = x.value();
        } catch (const std::exception &x) {
            e = py::reinterpret_borrow<py::object>(PyExc_ValueError)(x.what());
        }
        o.attr("fail")(e, slots);
    }
};

// The slot calls of a Python backend (InferenceSession(parallel=N) or a stub).
struct PySlotBackend {
    using Request = std::shared_ptr<PySlotRequest>;
    using Entry = py::object;
    py::object b;
    uint32_t slots() const { return b.attr("slots").cast<uint32_t>(); }
    uint32_t slotLen() const { return b.attr("slot_len").cast<uint32_t>(); }
    bool paged() const { return py::bool_(py::getattr(b, "paged", py::bool_(false))).cast<bool>(); }
    void slotPrefill(uint32_t slot, const std::vector<int32_t> &tokens, uint32_t pos) { b.attr("slot_prefill")(slot, tokens, pos); }
    void slotCopy(uint32_t src, uint32_t dst, uint32_t P) { b.attr("slot_copy")(src, dst, P); }
    void slotSampling(uint32_t slot, uint64_t seed, const Request &r) {
        const py::object &q = r->o;
        const py::object topK = q.attr("top_k"), minP = q.attr("min_p"), f = b.attr("slot_sampling");
        const auto args = py::make_tuple(slot, seed, q.attr("temperature"), q.attr("topp"), q.attr("presence"), q.attr("frequency"), q.attr("bias"));
        if (py::bool_(topK).cast<bool>() || py::bool_(minP).cast<bool>()) f(*args, py::arg("top_k") = topK, py::arg("min_p") = minP);
        else f(*args);
    }
    void slotLogprobs(uint32_t slot, int k) { b.attr("slot_logprobs")(slot, k); }
    std::vector<int32_t> slotsStep(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t active) {
        return b.attr("slots_step")(tokens, pos, activeList(active)).cast<std::vector<int32_t>>();
    }
    std::vector<int32_t> slotsStepLogprobs(const std::vector<int32_t> &tokens, const std::vector<int32_t> &pos, uint32_t active,
                                           std::vector<py::object> &entries) {
        const py::tuple r(b.attr("slots_step_logprobs")(tokens, pos, activeList(active)));
        entries = r[1].cast<std::vector<py::object>>();
        return r[0].cast<std::vector<int32_t>>();
    }
    bool slotReserve(uint32_t slot, uint32_t rows) { return py::bool_(b.attr("slot_reserve")(slot, rows)).cast<bool>(); }
    void slotTrim(uint32_t slot, uint32_t rows) { b.attr("slot_trim")(slot, rows); }
    void slotRelease(uint32_t slot) { b.attr("slot_release")(slot); }
    uint32_t freePages() const { return b.attr("free_pages")().cast<uint32_t>(); }
    uint32_t slotPageCount(uint32_t slot) const { return (uint32_t)py::len(b.attr("slot_pages")(slot)); }
    // Waits without the GIL. On the main thread, which alone receives signals, a pending signal's handler runs between slices and
    // its exception (KeyboardInterrupt) leaves run(). Another thread does not take the GIL back until a request comes, so that a
    // daemon thread never asks for it while the interpreter shuts down.
    template <class F> void asleep(const F &ready) const {
        const py::module_ threading = py::module_::import("threading");
        if (!threading.attr("current_thread")().is(threading.attr("main_thread")())) {
            py::gil_scoped_release nogil;
            while (!ready()) {}
            return;
        }
        while (true) {
            {
                py::gil_scoped_release nogil;
                if (ready()) return;
            }
            if (PyErr_CheckSignals() != 0) throw py::error_already_set();
        }
    }
private:
    std::vector<bool> activeList(uint32_t mask) const {
        std::vector<bool> a(slots());
        for (size_t i = 0; i < a.size(); i++) a[i] = (mask >> i) & 1u;
        return a;
    }
};
using PySlotScheduler = SlotScheduler<PySlotBackend>;
}  // namespace

PYBIND11_MODULE(_host, m) {
    m.doc() = "distributed_llama_b200 host library: .m/.t formats, q40/q80 codecs, TP slicers, tokenizer, sampler";

    // ---- quants ----
    m.attr("F_32") = (int)F_32;
    m.attr("F_16") = (int)F_16;
    m.attr("F_Q40") = (int)F_Q40;
    m.attr("F_Q80") = (int)F_Q80;
    m.def("parse_float_type", [](const std::string &s) { return (int)parseFloatType(s.c_str()); });
    m.def("float_type_name", [](int t) { return std::string(floatTypeName((FloatType)t)); });
    m.def("tensor_bytes", [](int t, size_t n) { return tensorBytes((FloatType)t, n); });
    m.def("f32_to_f16", &f32ToF16);
    m.def("f16_to_f32", &f16ToF32);
    m.def("quantize", [](int type, F32Array x) {
        const size_t n = (size_t)x.size();
        U8Array out((py::ssize_t)tensorBytes((FloatType)type, n));
        quantize((FloatType)type, x.data(), out.mutable_data(), n);
        return out;
    }, "Pack an f32 array into the byte stream of the given float type");
    m.def("dequantize", [](int type, U8Array in, size_t n) {
        if ((size_t)in.size() < tensorBytes((FloatType)type, n)) throw std::invalid_argument("dequantize: input too short");
        F32Array out((py::ssize_t)n);
        dequantize((FloatType)type, in.data(), out.mutable_data(), n);
        return out;
    });

    // ---- model format ----
    py::class_<ModelHeader>(m, "ModelHeader")
        .def(py::init<>())
        .def_readwrite("header_size", &ModelHeader::headerSize)
        .def_readwrite("file_size", &ModelHeader::fileSize)
        .def_readwrite("version", &ModelHeader::version)
        .def_property("arch", [](const ModelHeader &h) { return (int)h.arch; }, [](ModelHeader &h, int v) { h.arch = (ArchType)v; })
        .def_readwrite("dim", &ModelHeader::dim)
        .def_readwrite("hidden_dim", &ModelHeader::hiddenDim)
        .def_readwrite("moe_hidden_dim", &ModelHeader::moeHiddenDim)
        .def_readwrite("n_layers", &ModelHeader::nLayers)
        .def_readwrite("n_heads", &ModelHeader::nHeads)
        .def_readwrite("n_kv_heads", &ModelHeader::nKvHeads)
        .def_readwrite("head_dim", &ModelHeader::headDim)
        .def_readwrite("n_experts", &ModelHeader::nExperts)
        .def_readwrite("n_active_experts", &ModelHeader::nActiveExperts)
        .def_readwrite("vocab_size", &ModelHeader::vocabSize)
        .def_readwrite("seq_len", &ModelHeader::seqLen)
        .def_readwrite("orig_seq_len", &ModelHeader::origSeqLen)
        .def_readwrite("q_dim", &ModelHeader::qDim)
        .def_readwrite("kv_dim", &ModelHeader::kvDim)
        .def_property("hidden_act", [](const ModelHeader &h) { return (int)h.hiddenAct; }, [](ModelHeader &h, int v) { h.hiddenAct = (HiddenAct)v; })
        .def_property("rope_type", [](const ModelHeader &h) { return (int)h.ropeType; }, [](ModelHeader &h, int v) { h.ropeType = (RopeType)v; })
        .def_readwrite("rope_theta", &ModelHeader::ropeTheta)
        .def_readwrite("rope_scaling_factor", &ModelHeader::ropeScalingFactor)
        .def_readwrite("rope_scaling_low_freq_factor", &ModelHeader::ropeScalingLowFreqFactor)
        .def_readwrite("rope_scaling_high_freq_factor", &ModelHeader::ropeScalingHighFreqFactor)
        .def_readwrite("rope_scaling_orig_max_seq_len", &ModelHeader::ropeScalingOrigMaxSeqLen)
        .def_readwrite("norm_epsilon", &ModelHeader::normEpsilon)
        .def_property("weight_type", [](const ModelHeader &h) { return (int)h.weightType; }, [](ModelHeader &h, int v) { h.weightType = (FloatType)v; })
        .def_property_readonly("ff_dim", &ModelHeader::ffDim)
        .def_property_readonly("qk_norm", &ModelHeader::qkNorm)
        .def_property_readonly("arch_name", [](const ModelHeader &h) { return std::string(archName(h.arch)); })
        .def("describe", &describeModelHeader);
    m.attr("ARCH_LLAMA") = (int)ARCH_LLAMA;
    m.attr("ARCH_QWEN3") = (int)ARCH_QWEN3;
    m.attr("ARCH_QWEN3_MOE") = (int)ARCH_QWEN3_MOE;
    m.attr("ROPE_LLAMA") = (int)ROPE_LLAMA;
    m.attr("ROPE_FALCON") = (int)ROPE_FALCON;
    m.attr("ROPE_LLAMA3_1") = (int)ROPE_LLAMA3_1;
    m.attr("PART_ROOT") = (int)PART_ROOT;
    m.attr("PART_REPLICATE") = (int)PART_REPLICATE;
    m.attr("PART_ROWS") = (int)PART_ROWS;
    m.attr("PART_COLS") = (int)PART_COLS;
    m.def("load_model_header", &loadModelHeader, py::arg("path"), py::arg("max_seq_len") = 0);
    m.def("parse_model_header", [](py::bytes data, uint64_t fileSize, uint32_t maxSeqLen) {
        const std::string s = data;
        return parseModelHeader((const uint8_t *)s.data(), s.size(), fileSize, maxSeqLen);
    }, py::arg("data"), py::arg("file_size"), py::arg("max_seq_len") = 0);
    m.def("build_model_header", [](const std::vector<std::pair<int32_t, int32_t>> &kv) {
        const std::vector<uint8_t> b = buildModelHeader(kv);
        return py::bytes((const char *)b.data(), b.size());
    });

    py::class_<TensorEntry>(m, "TensorEntry")
        .def_readonly("name", &TensorEntry::name)
        .def_readonly("layer", &TensorEntry::layer)
        .def_readonly("expert", &TensorEntry::expert)
        .def_property_readonly("type", [](const TensorEntry &t) { return (int)t.type; })
        .def_readonly("d", &TensorEntry::d)
        .def_readonly("n", &TensorEntry::n)
        .def_readonly("offset", &TensorEntry::offset)
        .def_readonly("n_bytes", &TensorEntry::nBytes)
        .def_property_readonly("part", [](const TensorEntry &t) { return (int)t.part; })
        .def("__repr__", [](const TensorEntry &t) {
            return "<TensorEntry " + t.name + " L" + std::to_string(t.layer) + " E" + std::to_string(t.expert) + " " +
                   floatTypeName(t.type) + " [" + std::to_string(t.d) + "x" + std::to_string(t.n) + "] @" + std::to_string(t.offset) + ">";
        });
    py::class_<SliceRange>(m, "SliceRange")
        .def_readonly("first_row", &SliceRange::firstRow)
        .def_readonly("n_rows", &SliceRange::nRows)
        .def_readonly("row_bytes", &SliceRange::rowBytes)
        .def_readonly("col_byte_offset", &SliceRange::colByteOffset)
        .def_readonly("col_bytes", &SliceRange::colBytes)
        .def_readonly("first_col", &SliceRange::firstCol)
        .def_readonly("n_cols", &SliceRange::nCols)
        .def_property_readonly("total_bytes", &SliceRange::totalBytes);
    m.def("build_tensor_directory", &buildTensorDirectory, py::arg("header"), py::arg("check_file_size") = true);
    m.def("slice_tensor", &sliceTensor);
    m.def("extract_slice", [](const TensorEntry &t, py::buffer file, uint32_t rank, uint32_t nRanks) {
        py::buffer_info info = file.request();
        if ((uint64_t)info.size * (uint64_t)info.itemsize < t.offset + t.nBytes) throw std::invalid_argument("extract_slice: buffer too small");
        const SliceRange s = sliceTensor(t, rank, nRanks);
        U8Array out((py::ssize_t)s.totalBytes());
        extractSlice(t, (const uint8_t *)info.ptr, rank, nRanks, out.mutable_data());
        return out;
    });
    m.def("build_rope_table", [](const ModelHeader &h, uint32_t seqLen) {
        py::array_t<float> out({(py::ssize_t)seqLen, (py::ssize_t)(h.headDim / 2), (py::ssize_t)2});
        buildRopeTable(h, seqLen, out.mutable_data());
        return out;
    });
    m.def("rope_frequency", &ropeFrequency);
    m.def("required_device_bytes", &requiredDeviceBytes);

    // ---- text ----
    py::class_<TokenizerData>(m, "TokenizerData")
        .def(py::init<>())
        .def_property("vocab",
            [](const TokenizerData &d) { py::list l; for (auto &t : d.vocab) l.append(asBytes(t)); return l; },
            [](TokenizerData &d, const std::vector<py::bytes> &v) { d.vocab.clear(); for (auto &b : v) d.vocab.push_back((std::string)b); })
        .def_readwrite("scores", &TokenizerData::scores)
        .def_readwrite("bos_id", &TokenizerData::bosId)
        .def_readwrite("add_bos", &TokenizerData::addBos)
        .def_readwrite("eos_ids", &TokenizerData::eosIds)
        .def_property("chat_template",
            [](const TokenizerData &d) { return asBytes(d.chatTemplate); },
            [](TokenizerData &d, py::bytes b) { d.chatTemplate = (std::string)b; })
        .def_readwrite("max_token_length", &TokenizerData::maxTokenLength);
    m.def("read_tokenizer_file", &readTokenizerFile);
    m.def("write_tokenizer_file", &writeTokenizerFile);

    py::class_<Tokenizer>(m, "Tokenizer")
        .def(py::init<const std::string &>())
        .def(py::init<TokenizerData>())
        .def("encode", [](const Tokenizer &t, py::object text, bool isStart, bool addSpecial) {
            std::string s = py::isinstance<py::bytes>(text) ? (std::string)text.cast<py::bytes>() : text.cast<std::string>();
            return t.encode(s, isStart, addSpecial);
        }, py::arg("text"), py::arg("is_start") = true, py::arg("add_special_tokens") = true)
        .def("decode", [](Tokenizer &t, int32_t token) { return asBytes(t.decode(token)); })
        .def("reset_decoder", &Tokenizer::resetDecoder)
        .def("is_eos", &Tokenizer::isEos)
        .def("describe", &Tokenizer::describe)
        .def("piece", [](const Tokenizer &t, int32_t id) { return asBytes(t.data().vocab.at(id)); })
        .def_property_readonly("vocab_size", &Tokenizer::vocabSize)
        .def_property_readonly("regular_vocab_size", &Tokenizer::regularVocabSize)
        .def_property_readonly("bos_id", [](const Tokenizer &t) { return t.data().bosId; })
        .def_property_readonly("add_bos", [](const Tokenizer &t) { return t.data().addBos; })
        .def_property_readonly("eos_ids", [](const Tokenizer &t) { return t.data().eosIds; })
        .def_property_readonly("chat_template", [](const Tokenizer &t) { return asBytes(t.data().chatTemplate); });

    // Streaming decoder state of one sequence over a shared tokenizer (the choices of one request each keep their own).
    struct TokenDecoder { std::string pending; };
    py::class_<TokenDecoder>(m, "TokenDecoder")
        .def(py::init<>())
        .def("decode", [](TokenDecoder &d, const Tokenizer &t, int32_t token) { return asBytes(t.decodeWith(d.pending, token)); })
        .def("reset", [](TokenDecoder &d) { d.pending.clear(); });
    m.def("choice_seed", &choiceSeed, py::arg("seed"), py::arg("index"));

    py::class_<PySlotScheduler>(m, "SlotScheduler")
        .def(py::init([](py::object backend, py::object seedSource, py::object onEvict) {
            std::function<void(uint32_t)> evict;
            if (!onEvict.is_none()) evict = [onEvict](uint32_t s) { onEvict(s); };
            return new PySlotScheduler(PySlotBackend{std::move(backend)}, [seedSource] { return seed64(seedSource()); }, evict);
        }), py::arg("backend"), py::arg("seed_source"), py::arg("on_evict") = py::none())
        .def("submit", [](PySlotScheduler &s, py::object req) { s.submit(std::make_shared<PySlotRequest>(PySlotRequest{std::move(req)})); })
        .def("stop", &PySlotScheduler::stop)
        .def("run", &PySlotScheduler::run);

    py::class_<Rng>(m, "Rng")
        .def(py::init<uint64_t>())
        .def("next_u32", &Rng::nextU32)
        .def("next_f32", &Rng::nextF32)
        .def_readwrite("state", &Rng::state);

    py::class_<Sampler>(m, "Sampler")
        .def(py::init<uint32_t, float, float, uint64_t>())
        .def("sample", [](Sampler &s, F32Array logits) {
            if ((uint32_t)logits.size() < s.vocabSize()) throw std::invalid_argument("Sampler: logits shorter than vocab size");
            F32Array copy = logits.attr("copy")().cast<F32Array>();
            return s.sample(copy.mutable_data());
        })
        .def("set_controls", [](Sampler &s, float presence, float frequency, const std::vector<std::pair<int32_t, float>> &bias) {
            s.setControls(presence, frequency, bias);
        }, py::arg("presence_penalty"), py::arg("frequency_penalty"), py::arg("logit_bias") = std::vector<std::pair<int32_t, float>>{})
        .def("set_filters", &Sampler::setFilters, py::arg("top_k"), py::arg("min_p"))
        .def_property_readonly("top_k", &Sampler::topK)
        .def_property_readonly("min_p", &Sampler::minP)
        .def_property_readonly("filters_active", &Sampler::filtersActive)
        .def("begin_completion", &Sampler::beginCompletion)
        .def("apply_controls", [](const Sampler &s, F32Array logits) {
            if ((uint32_t)logits.size() < s.vocabSize()) throw std::invalid_argument("Sampler: logits shorter than vocab size");
            F32Array copy = logits.attr("copy")().cast<F32Array>();
            s.applyControls(copy.mutable_data());
            return copy;
        })
        .def_property_readonly("controls_active", &Sampler::controlsActive)
        .def_property_readonly("presence_penalty", &Sampler::presencePenalty)
        .def_property_readonly("frequency_penalty", &Sampler::frequencyPenalty)
        .def_property_readonly("logit_bias", &Sampler::logitBias)
        .def_property_readonly("counts", [](const Sampler &s) {
            const std::vector<uint32_t> &c = s.counts();
            return py::array_t<uint32_t>((py::ssize_t)c.size(), c.data());
        })
        .def_property_readonly("completion_generation", &Sampler::completionGeneration)
        .def("next_coin", &Sampler::nextCoin)
        .def("next_seed", &Sampler::nextSeed)
        .def("set_temperature", &Sampler::setTemperature)
        .def("set_topp", &Sampler::setTopp)
        .def("set_seed", &Sampler::setSeed)
        .def_property_readonly("seed", &Sampler::seed)
        .def_property_readonly("seed_generation", &Sampler::seedGeneration)
        .def_property_readonly("temperature", &Sampler::temperature)
        .def_property_readonly("topp", &Sampler::topp)
        .def_property_readonly("vocab_size", &Sampler::vocabSize);
    m.def("softmax", [](F32Array x) {
        F32Array out = x.attr("copy")().cast<F32Array>();
        softmaxInPlace(out.mutable_data(), (size_t)out.size());
        return out;
    });

    m.attr("TEMPLATE_UNKNOWN") = (int)TEMPLATE_UNKNOWN;
    m.attr("TEMPLATE_LLAMA2") = (int)TEMPLATE_LLAMA2;
    m.attr("TEMPLATE_LLAMA3") = (int)TEMPLATE_LLAMA3;
    m.attr("TEMPLATE_DEEP_SEEK3") = (int)TEMPLATE_DEEP_SEEK3;
    m.attr("TEMPLATE_CHATML") = (int)TEMPLATE_CHATML;
    m.def("parse_chat_template_type", [](const std::string &s) { return (int)parseChatTemplateType(s); });
    py::class_<ChatTemplateGenerator>(m, "ChatTemplateGenerator")
        .def(py::init([](int type, py::bytes tpl, py::bytes eos) {
            return new ChatTemplateGenerator((ChatTemplateType)type, (std::string)tpl, (std::string)eos);
        }))
        .def("generate", [](const ChatTemplateGenerator &g, const std::vector<std::pair<std::string, std::string>> &items, bool gen) {
            std::vector<ChatItem> v;
            for (auto &p : items) v.push_back({p.first, p.second});
            GeneratedChat c = g.generate(v, gen);
            return py::make_tuple(asBytes(c.content), asBytes(c.publicPrompt));
        }, py::arg("items"), py::arg("append_generation_prompt") = true)
        .def_property_readonly("type", [](const ChatTemplateGenerator &g) { return (int)g.type(); })
        .def_property_readonly("type_name", [](const ChatTemplateGenerator &g) { return std::string(chatTemplateTypeName(g.type())); });

    m.attr("MAYBE_EOS") = (int)MAYBE_EOS;
    m.attr("EOS") = (int)EOS;
    m.attr("NOT_EOS") = (int)NOT_EOS;
    py::class_<EosDetector>(m, "EosDetector")
        .def(py::init([](std::vector<int32_t> tokens, const std::vector<py::bytes> &pieces, int padLeft, int padRight) {
            std::vector<std::string> p;
            for (auto &b : pieces) p.push_back((std::string)b);
            return new EosDetector(std::move(tokens), std::move(p), padLeft, padRight);
        }))
        .def("append", [](EosDetector &d, int32_t tokenId, py::object piece) {
            std::string s;
            if (!piece.is_none()) s = py::isinstance<py::bytes>(piece) ? (std::string)piece.cast<py::bytes>() : piece.cast<std::string>();
            return (int)d.append(tokenId, s);
        })
        .def("is_eos", &EosDetector::isEos)
        .def("get_delta", [](const EosDetector &d) { return asBytes(d.getDelta()); })
        .def("reset", &EosDetector::reset);

    m.attr("MAX_STOP_STRINGS") = kMaxStopStrings;
    m.attr("MAX_STOP_BYTES") = kMaxStopBytes;
    py::class_<StopMatcher>(m, "StopMatcher")
        .def(py::init([](const std::vector<py::bytes> &stops) {
            std::vector<std::string> s;
            for (auto &b : stops) s.push_back((std::string)b);
            return new StopMatcher(std::move(s));
        }))
        .def("push", [](StopMatcher &s, py::bytes delta) { return asBytes(s.push((std::string)delta)); })
        .def("flush", [](StopMatcher &s) { return asBytes(s.flush()); })
        .def_property_readonly("stopped", &StopMatcher::stopped)
        .def_property_readonly("held", [](const StopMatcher &s) { return asBytes(s.held()); });
}
