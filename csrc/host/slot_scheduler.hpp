// The scheduler of concurrent requests on KV-cache slots (`--parallel`), the one both API servers run: ApiServer::serveParallel
// over InferenceBackend (csrc/app/api_server.cpp), distributed_llama_b200.api.SlotScheduler over Python objects (bindings.cpp).
//
// One engine thread (run) owns the GPU and decodes every busy slot in one batched step per token.
//
// Between steps it admits waiting requests first-in, first-out into free slots: a request takes n slots (one when greedy: every
// greedy completion is the same), the free slot whose prompt cache covers most of its messages first (lowest index on ties). It
// prefills the request's delta prompt into that slot (the running rows wait for this prefill), copies the prompt rows into its
// other slots and seeds each slot: completion i with choiceSeed(seed, i) when n > 1, the seed itself when n = 1; a request
// without a seed takes seedSource() in admission order. The prompt's last token then enters the next batched step. A completion
// stops at end of sequence or after min(maxTokens, slotLen - P) tokens. If a hook throws (a client went away), the request ends
// and frees its slots; the other requests continue. A request for more completions than there are slots fails at submit.
//
// Paged slots (paged(): the slots share the KV cache as one pool of 64-row pages): a request is admitted, still first in, first
// out, only when every slot it takes can hold rows [0, P + 64) (P = promptLen(slot), capped at slotLen); otherwise it and
// everything behind it wait. Each slot it takes keeps exactly the pages of those rows: pages a previous occupant left beyond them
// go back to the pool (the rows it reuses, [0, P), lie inside). A running row reserves its next page when its position reaches
// a page boundary. A finished slot keeps its pages as its prompt cache; when an admission or a growing row needs pages, idle
// slots' caches are evicted whole, least recently finished first (slotRelease, then onEvict(slot): the server forgets that slot's
// prompt cache). A row that cannot get a page ends there, as if it had reached its length limit. A request that needs more pages
// than the pool holds fails. The slots of a request that fails give their pages back.
//
// Backend: the types Request (a shared_ptr to a request) and Entry (one row's log-probabilities, passed on untouched), the slot
// calls of InferenceBackend (paged only: slotReserve, slotTrim, slotRelease, freePages, slotPageCount) with slotSampling(slot,
// seed, request) setting up the request's sampling, and asleep(ready), which calls ready() until it returns true: each call waits
// up to kSlotWaitSlice for a request (Python: without the GIL; on the main thread a signal such as Ctrl-C ends run between calls).
// Request: n(), greedy(), seed() (empty: none), maxTokens() (<= 0: none), logprobs() (-1: none) and the hooks of
// distributed_llama_b200.api.SlotRequest.
// submit and stop may be called from any thread, run from one; no hook or backend call is made under the queue lock. What a hook
// or an admission's backend call throws goes to the request's fail; what the step or page growth throws leaves run.
#pragma once
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <exception>
#include <functional>
#include <memory>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "text.hpp"

namespace dl {

constexpr uint32_t kSlotPageRows = 64;   // rows of a KV-cache page (csrc/cuda/engine.cu)
constexpr std::chrono::milliseconds kSlotWaitSlice{100};   // an idle run() wakes this often (Python: to see signals)

// A prompt resolved against a slot's cache: the tokens to prefill from `start`, the last prompt token and its position P.
struct SlotPrompt {
    std::vector<int32_t> prefill;
    uint32_t start = 0;
    int32_t token = 0;
    uint32_t P = 0;
};

template <class Backend>
class SlotScheduler {
public:
    using Request = typename Backend::Request;
    using Entry = typename Backend::Entry;

    SlotScheduler(Backend backend, std::function<uint64_t()> seedSource, std::function<void(uint32_t)> onEvict = nullptr)
        : be_(std::move(backend)), seedSource_(std::move(seedSource)), onEvict_(std::move(onEvict)), N_(be_.slots()), L_(be_.slotLen()),
          paged_(be_.paged()), rows_(N_), finished_(N_, 0) {}

    // Queues the request; one for no completions or for more completions than there are slots is refused at once.
    void submit(Request req) {
        const uint32_t n = req->n();
        if (n < 1 || rowsOf(req) > N_) {
            const std::string why = n < 1 ? "n must be at least 1" : "n = " + std::to_string(n) + " needs more than the " + std::to_string(N_) + " slots";
            req->fail(std::make_exception_ptr(std::invalid_argument(why)), {});
            return;
        }
        std::lock_guard<std::mutex> lk(mu_);
        queue_.push_back(std::move(req));
        cv_.notify_all();
    }

    // run returns before its next step.
    void stop() {
        std::lock_guard<std::mutex> lk(mu_);
        stopped_ = true;
        cv_.notify_all();
    }

    void run() {
        std::deque<Request> waiting;
        const auto running = [&](const Row &r) { return r.left > 0; };
        while (take(waiting, waiting.empty() && std::none_of(rows_.begin(), rows_.end(), running))) {
            while (!waiting.empty()) {
                std::vector<uint32_t> free;
                for (uint32_t s = 0; s < N_; s++) if (!rows_[s].job) free.push_back(s);
                if (free.size() < rowsOf(waiting.front()) || !admit(waiting.front(), free)) break;
                waiting.pop_front();
            }
            if (paged_) grow();
            std::vector<int32_t> tokens(N_, 0), pos(N_, 0);
            uint32_t active = 0;
            bool wantLp = false;
            for (uint32_t s = 0; s < N_; s++) {
                if (!rows_[s].left) continue;
                tokens[s] = rows_[s].token;
                pos[s] = rows_[s].pos;
                active |= 1u << s;
                wantLp = wantLp || rows_[s].job->logprobs;
            }
            if (!active) continue;
            std::vector<Entry> entries;
            const std::vector<int32_t> drawn = wantLp ? be_.slotsStepLogprobs(tokens, pos, active, entries) : be_.slotsStep(tokens, pos, active);
            for (uint32_t s = 0; s < N_; s++) {
                Row &r = rows_[s];
                if (!r.left) continue;
                const std::shared_ptr<Job> job = r.job;
                r.token = drawn[s];
                r.pos++;
                try {
                    for (uint32_t i = r.first; i < r.first + r.count; i++) {
                        if (job->done[i]) continue;
                        job->out[i].push_back(drawn[s]);
                        if (job->logprobs) job->req->onLogprobs(i, entries.at(s));
                        if (job->req->onToken(i, drawn[s]) || (int64_t)job->out[i].size() >= job->limit) { job->done[i] = true; r.left--; }
                    }
                } catch (...) {
                    release(*job);
                    fail(job->req, job->slots, std::current_exception());
                    continue;
                }
                if (!r.left) rowDone(s);
            }
        }
    }

private:
    // An admitted request: its slots, P, length limit, rows still running and its completions' tokens.
    struct Job {
        Request req;
        std::vector<uint32_t> slots;
        uint32_t P, live;
        int64_t limit;
        bool logprobs;
        std::vector<std::vector<int32_t>> out;
        std::vector<bool> done;
    };
    // A slot's owner and, while it runs (left > 0), the token it feeds at `pos` and the completions [first, first + count) it
    // serves (all n of a greedy request, else one), `left` of them unfinished.
    struct Row {
        std::shared_ptr<Job> job;
        int32_t token = 0, pos = 0;
        uint32_t first = 0, count = 0, left = 0;
    };

    static uint32_t rowsOf(const Request &req) { return req->greedy() ? 1 : req->n(); }

    // Moves what was submitted into `waiting`; block: sleeps until something is. False once stop() was called.
    bool take(std::deque<Request> &waiting, bool block) {
        const auto ready = [&] { return !queue_.empty() || stopped_; };
        if (block) be_.asleep([&] {
            std::unique_lock<std::mutex> lk(mu_);
            return cv_.wait_for(lk, kSlotWaitSlice, ready);
        });
        std::lock_guard<std::mutex> lk(mu_);
        for (Request &r : queue_) waiting.push_back(std::move(r));
        queue_.clear();
        return !stopped_;
    }

    // Evicts idle caches, least recently finished first and none of `keep`, until `pages` pages are free; false (nothing evicted)
    // if even all of them would not do.
    bool evictFor(int64_t pages, const std::vector<uint32_t> &keep) {
        std::vector<uint32_t> idle;
        int64_t avail = be_.freePages();
        for (uint32_t s = 0; s < N_; s++) {
            if (rows_[s].job || std::find(keep.begin(), keep.end(), s) != keep.end()) continue;
            const uint32_t n = be_.slotPageCount(s);
            if (n > 0) { idle.push_back(s); avail += n; }
        }
        if (avail < pages) return false;
        std::stable_sort(idle.begin(), idle.end(), [&](uint32_t a, uint32_t b) { return finished_[a] < finished_[b]; });
        for (uint32_t s : idle) {
            if (be_.freePages() >= pages) break;
            be_.slotRelease(s);
            if (onEvict_) onEvict_(s);
        }
        return true;
    }

    static uint32_t pagesOf(uint32_t rows) { return (rows + kSlotPageRows - 1) / kSlotPageRows; }

    // Starts `req` in free slots; false when paged slots cannot reserve its pages yet (nothing changed).
    bool admit(const Request &req, const std::vector<uint32_t> &free) {
        uint32_t first = free[0];
        size_t best = req->cachedPrefix(first);
        for (size_t k = 1; k < free.size(); k++) {
            const size_t n = req->cachedPrefix(free[k]);
            if (n > best) { best = n; first = free[k]; }
        }
        std::vector<uint32_t> slots{first};
        for (uint32_t s : free) if (s != first && slots.size() < rowsOf(req)) slots.push_back(s);
        try {
            if (paged_) {
                const uint32_t want = std::min(L_, req->promptLen(first) + kSlotPageRows), pages = pagesOf(want) * (uint32_t)slots.size();
                if (pages > L_ / kSlotPageRows)
                    throw std::invalid_argument("the request needs " + std::to_string(pages) + " KV-cache pages, more than the pool's " +
                                                std::to_string(L_ / kSlotPageRows));
                int64_t net = pages;   // free pages the admission takes once its slots give back what they hold beyond `want`
                for (uint32_t s : slots) net -= be_.slotPageCount(s);
                if (!evictFor(net, slots)) return false;
                for (uint32_t s : slots) be_.slotTrim(s, want);
                for (uint32_t s : slots) be_.slotReserve(s, want);   // cannot fail: the pages are free
            }
            start(req, slots);
        } catch (...) {   // e.g. the client went away while its prompt was prepared
            fail(req, slots, std::current_exception());
        }
        return true;
    }

    void start(const Request &req, const std::vector<uint32_t> &slots) {
        const SlotPrompt p = req->prepare(slots[0]);
        if (!p.prefill.empty()) be_.slotPrefill(slots[0], p.prefill, p.start);
        for (size_t k = 1; k < slots.size(); k++) be_.slotCopy(slots[0], slots[k], p.P);
        const std::optional<uint64_t> given = req->seed();
        const uint64_t seed = given ? *given : (req->greedy() ? 0 : seedSource_());
        const uint32_t n = req->n();
        const int lp = req->logprobs();
        for (uint32_t k = 0; k < slots.size(); k++) {
            be_.slotSampling(slots[k], n == 1 ? seed : choiceSeed(seed, k), req);
            if (lp >= 0) be_.slotLogprobs(slots[k], lp);
        }
        const int64_t room = (int64_t)L_ - p.P, limit = req->maxTokens() > 0 ? std::min(room, req->maxTokens()) : room;
        const auto job = std::make_shared<Job>(Job{req, slots, p.P, (uint32_t)slots.size(), limit, lp >= 0,
                                                   std::vector<std::vector<int32_t>>(n), std::vector<bool>(n, false)});
        if (limit <= 0) { req->finish(job->out, slots, p.P); return; }
        for (uint32_t k = 0; k < slots.size(); k++) {
            const bool all = slots.size() == 1;
            rows_[slots[k]] = Row{job, p.token, (int32_t)p.P, all ? 0 : k, all ? n : 1, all ? n : 1};
        }
    }

    void release(const Job &job) {
        for (uint32_t s : job.slots)
            if (rows_[s].job.get() == &job) { rows_[s] = Row(); finished_[s] = ++clock_; }
    }

    // The request ends early; its slots' rows may not match a prompt cache, so paged slots give their pages back.
    void fail(const Request &req, const std::vector<uint32_t> &slots, std::exception_ptr error) {
        if (paged_) for (uint32_t s : slots) be_.slotRelease(s);
        req->fail(error, slots);
    }

    // Slot s's row has finished every completion it serves; the request finishes with its last row.
    void rowDone(uint32_t s) {
        const std::shared_ptr<Job> job = rows_[s].job;
        rows_[s].left = 0;
        if (--job->live > 0) return;
        release(*job);
        try { job->req->finish(job->out, job->slots, job->P); } catch (...) { fail(job->req, job->slots, std::current_exception()); }
    }

    // Paged: every row about to write a row past its pages reserves the next page (evicting idle caches); one that cannot ends.
    void grow() {
        for (uint32_t s = 0; s < N_; s++) {
            if (!rows_[s].left) continue;
            const uint32_t rows = (uint32_t)rows_[s].pos + 1;
            const int64_t shortPages = (int64_t)pagesOf(rows) - be_.slotPageCount(s);
            if (shortPages <= 0) continue;
            std::vector<uint32_t> busy;
            for (uint32_t t = 0; t < N_; t++) if (rows_[t].left) busy.push_back(t);
            if (!evictFor(shortPages, busy) || !be_.slotReserve(s, rows)) rowDone(s);
        }
    }

    Backend be_;
    const std::function<uint64_t()> seedSource_;
    const std::function<void(uint32_t)> onEvict_;
    const uint32_t N_, L_;
    const bool paged_;
    std::vector<Row> rows_;
    std::vector<uint64_t> finished_;   // paged: when each slot's cache was last left idle (eviction order)
    uint64_t clock_ = 0;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<Request> queue_;
    bool stopped_ = false;
};

}  // namespace dl
