"""Public Python API: load a `.m`/`.t` pair and run inference on the local rank(s).

    from distributed_llama_b200.api import InferenceSession
    s = InferenceSession("model.m", "tokenizer.t")
    text = s.generate("Hello", steps=64)

This is the call path `dllama inference|chat|perplexity` and `dllama-api` sit on (reference: runInferenceApp,
src/app.cpp:232-304).
"""
from __future__ import annotations

import os
import time
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import host
from .formats.model_file import ModelFile
from .ops.cuda_lib import SLOT_CACHE_LAYOUTS
from .parallel.control import (OP_CHOICES_FIRST, OP_CHOICES_SEED, OP_CHOICES_STEP, OP_CONTROLS, OP_DECODE_N, OP_FILTERS, OP_PREFILL,
                               OP_SEED, OP_STEP_GREEDY, OP_STEP_LOGITS, OP_STEP_SAMPLE, _active_mask, _f32_bits, _split_seed)


@dataclass
class GenerationStats:
    n_prompt_tokens: int = 0
    n_generated: int = 0
    prefill_ms: float = 0.0
    decode_ms: float = 0.0


MAX_CHOICES = 8   # the engine's widest batch: one row per choice
MAX_TOP_LOGPROBS = 20   # the largest `top_logprobs` (csrc/cuda/logprobs.cu)


def check_logprobs(k: int, n_ranks: int = 1) -> None:
    """Raises ValueError unless log-probabilities with k top entries can run here: 0 <= k <= 20, one GPU (under tensor
    parallelism the vocabulary is sliced over the ranks)."""
    if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k <= MAX_TOP_LOGPROBS:
        raise ValueError(f"top_logprobs must be an integer from 0 to {MAX_TOP_LOGPROBS}")
    if n_ranks > 1:
        raise ValueError("logprobs are not supported under tensor parallelism yet")


MAX_STOP_STRINGS = 4   # a request's `stop` strings, each of 1 to MAX_STOP_BYTES bytes (host StopMatcher)
MAX_STOP_BYTES = 256


def check_stop(stop) -> List[bytes]:
    """Stop strings as the UTF-8 bytes a host StopMatcher matches: None and [] mean none, else a string or a list of at most 4
    strings of 1 to 256 bytes each. Anything else raises ValueError, as does a string with an unpaired surrogate."""
    if stop is None:
        return []
    items = [stop] if isinstance(stop, str) else stop
    if not isinstance(items, list) or len(items) > MAX_STOP_STRINGS or not all(isinstance(s, str) for s in items):
        raise ValueError(f"'stop' must be a string or an array of at most {MAX_STOP_STRINGS} strings")
    out = []
    for s in items:
        try:
            b = s.encode("utf-8")
        except UnicodeEncodeError:
            raise ValueError("'stop' strings must not hold unpaired surrogates") from None
        if not 1 <= len(b) <= MAX_STOP_BYTES:
            raise ValueError(f"'stop' strings must be 1 to {MAX_STOP_BYTES} bytes long")
        out.append(b)
    return out


def run_choices(backend, token: int, P: int, n: int, max_tokens: int, seq_len: int, sampler, base_seed: int,
                on_token: Callable[[int, int], bool], logprobs: Optional[int] = None,
                on_logprobs: Optional[Callable[[int, tuple], None]] = None) -> List[List[int]]:
    """Generates n completions of one prompt whose last token `token` sits at position P, everything before it prefilled.

    Choice i draws with an xorshift* generator seeded with choice_seed(base_seed, i); its j-th token has rotary position
    P + 1 + j and its K/V row is P + 1 + i*C + j with C = (seq_len - 1 - P) // n, so the choices share the rest of the context
    window and each stops after min(max_tokens, C) tokens (max_tokens <= 0: C). A single completion (n = 1) is the
    single-sequence loop of `generate` and the CLIs instead: it stops after min(max_tokens, seq_len - P) tokens, so it may fill
    the context up to its last row. Rows up to P-1 are never written; row P is written by the forward
    of `token` (once on the batched path, once per choice, with the same values, on the sequential path). The single-sequence
    generator continues its stream afterwards. on_token(i, tok) is called for every generated token and returns True when
    choice i is finished (end of sequence or stop string). The sampler's controls (presence / frequency penalty, logit bias)
    apply to every choice, each with its own token counts, which start at zero, and so do its filters (top_k, min_p; the
    backend's choice_controls hands them to the batched path). `backend` provides
    next_token(token, pos, sampler), forget_device_seed(), save_sampler() / restore_sampler(saved), and for the batched path
    batched_choices(n), seed_choices(seeds), choice_controls(sampler, n), choices_first(token, P, n, T, topp) and
    choices_step(tokens, P, C, j, active, T, topp) (TokenSteps: InferenceSession and apps.runtime.RootInference), and with a draft
    model (backend.draft set) speculates(sampler) and spec_round(token, pos). Returns each choice's tokens.

    logprobs = k (0..20): on_logprobs(i, entry) is called right before on_token(i, tok) with the entry of that token,
    (tok, logprob, [(id, logprob), ...] k most likely); the backend's next_token, choices_first and choices_step then take a
    `logprobs=k` keyword and last_logprobs() returns the entries of their last call, one per row. The tokens are the same as
    without it."""
    H = host()
    if not 1 <= n <= MAX_CHOICES:
        raise ValueError(f"n must be between 1 and {MAX_CHOICES}")
    lp = {} if logprobs is None else {"logprobs": logprobs}
    C = (seq_len - 1 - P) // n
    limit = seq_len - P if n == 1 else C
    if max_tokens > 0:
        limit = min(max_tokens, limit)
    out: List[List[int]] = [[] for _ in range(n)]
    if limit <= 0:
        return out
    sampler.begin_completion()

    def single(smp, choices):
        # today's single-sequence path from P; rows past P belong to this sequence until the next one overwrites them. A single
        # greedy completion with a draft model takes speculative rounds of several tokens instead (the same tokens).
        tok, pos, done = token, P, set()
        spec = n == 1 and not lp and getattr(backend, "draft", None) is not None and backend.speculates(smp)
        while len(out[choices[0]]) < limit:
            toks = backend.spec_round(tok, pos) if spec else [backend.next_token(tok, pos, smp, **lp)]
            entry = backend.last_logprobs()[0] if lp else None
            for tok in toks:
                pos += 1
                for i in choices:
                    if i not in done:
                        out[i].append(tok)
                        if lp:
                            on_logprobs(i, entry)
                        if on_token(i, tok):
                            done.add(i)
                if len(done) == len(choices) or len(out[choices[0]]) >= limit:
                    break
            if len(done) == len(choices):
                break

    if n == 1 or sampler.temperature == 0.0:
        # greedy choices are all equal: one run
        single(sampler, list(range(n)))
        return out
    T, topp = sampler.temperature, sampler.topp
    seeds = [H.choice_seed(base_seed, i) for i in range(n)]
    if not backend.batched_choices(n):
        saved = backend.save_sampler()
        try:
            for i in range(n):
                backend.forget_device_seed()
                smp = H.Sampler(sampler.vocab_size, T, topp, seeds[i])   # a fresh sampler: its own counts, from zero
                smp.set_controls(sampler.presence_penalty, sampler.frequency_penalty, sampler.logit_bias)
                smp.set_filters(sampler.top_k, sampler.min_p)
                single(smp, [i])
        finally:
            backend.restore_sampler(saved)
        return out
    backend.seed_choices(seeds)
    backend.choice_controls(sampler, n)
    last = backend.choices_first(token, P, n, T, topp, **lp)
    active = [True] * n
    j = 0
    while True:
        entries = backend.last_logprobs() if lp else None
        for i in range(n):
            if active[i]:
                out[i].append(last[i])
                if lp:
                    on_logprobs(i, entries[i])
                if on_token(i, last[i]) or len(out[i]) >= limit:
                    active[i] = False
        if not any(active):
            break
        last = backend.choices_step(last, P, C, j, active, T, topp, **lp)
        j += 1
    return out


def _lp_kw(logprobs: Optional[int]) -> dict:
    """The engine's `logprobs` keyword, passed only when log-probabilities are asked for."""
    return {} if logprobs is None else {"logprobs": logprobs}


class SpecStats:
    """Counters of speculative rounds: rounds, drafted and accepted tokens, emitted tokens."""

    def __init__(self):
        self.rounds = self.drafted = self.accepted = self.emitted = 0

    def add(self, drafted: int, accepted: int, emitted: int) -> None:
        self.rounds += 1
        self.drafted += drafted
        self.accepted += accepted
        self.emitted += emitted

    def line(self) -> str:
        """The CLIs' summary line."""
        rate = 100.0 * self.accepted / self.drafted if self.drafted else 0.0
        per = self.emitted / self.rounds if self.rounds else 0.0
        return (f"Speculative: {self.rounds} rounds, {self.drafted} drafted, {self.accepted} accepted ({rate:.1f} %), "
                f"{per:.2f} tokens/round")


DRAFT_TOKENS = (1, 3, 7)   # --draft-tokens: the verify forward runs k + 1 rows, a power of two


class DraftRefused(ValueError):
    """A --draft-model setting this configuration cannot run (see draft_refusal)."""


def draft_refusal(draft_tokens: int, n_ranks: int = 1, parallel: int = 1, headers: Sequence = ()) -> Optional[str]:
    """Why greedy speculative decoding with a draft model of `draft_tokens` drafts per round cannot run here, or None if it can.
    headers: (name, model header) of the target and the draft, checked once they are read (the draft's with the target's context
    length: a shorter draft context is refused)."""
    if draft_tokens not in DRAFT_TOKENS:
        return "--draft-tokens must be 1, 3 or 7"
    if n_ranks > 1:
        return "--draft-model runs on one GPU only (no --gpus > 1 or --workers)"
    if os.environ.get("DL_COLLECTIVES") == "nccl":
        return "--draft-model does not support DL_COLLECTIVES=nccl"
    if parallel > 1:
        return "--draft-model does not combine with --parallel > 1"
    H = host() if headers else None
    for name, h in headers:
        if h.n_experts > 0:
            return f"--draft-model needs dense models: the {name} is mixture-of-experts (no batched verify step)"
        if h.weight_type != H.F_Q40:
            return f"--draft-model needs q40 weights: the {name} has {H.float_type_name(h.weight_type)} weights"
    if len(headers) == 2:
        t, d = headers[0][1], headers[1][1]
        if t.vocab_size != d.vocab_size:
            return f"--draft-model needs the target's vocabulary: {t.vocab_size} tokens against {d.vocab_size}"
        if d.seq_len < t.seq_len:
            return f"--draft-model needs a context of at least {t.seq_len} tokens: the draft model has {d.seq_len}"
    return None


class TokenSteps:
    """The token steps of one engine, the backend run_choices needs: InferenceSession for the library and
    apps.runtime.RootInference for the CLIs and API server, which announces every engine call to the workers (_send).

    Greedy draws without sampling controls run on the fused arg-max. Other draws run on the device sampler
    (csrc/cuda/sampler.cu: the logits never leave the GPUs), unless the engine is not on a GPU, its collectives are the
    library's (multi-node) or DL_HOST_SAMPLER is set: then the host sampler draws from logits copied back. The device's
    generator, controls and filters are handed over when the sampler's differ from what the device holds."""

    def __init__(self, engine, device, n_ranks: int, draft=None, draft_tokens: int = 3):
        self.engine = engine
        self.device = torch.device(device)
        self.n_ranks = n_ranks
        self.draft = draft                  # runtime.engine.Engine of the draft model, or None (speculates)
        self.draft_tokens = draft_tokens
        self.spec_stats = SpecStats()
        # the caller synchronises every step, so one pinned staging slot is enough (workers enqueue ahead: pageable staging)
        on_gpu = self.device.type == "cuda"
        self._pin_in = torch.zeros(2, dtype=torch.int32).pin_memory() if on_gpu else None
        self._pin_out = torch.zeros(1, dtype=torch.int32).pin_memory() if on_gpu else None
        self._dev_seeded = None          # (seed, seed generation) of the sampler the device generator follows (None: none)
        self._dev_controls = None        # completion generation whose controls the device holds (None: off)
        self._dev_filters = (0, 0.0)     # (top_k, min_p) the device holds
        self._last_logprobs = None

    def _send(self, op: int, pos: int, words: Sequence[int]) -> None:
        """Announces an engine call every worker must repeat (parallel.control packets); no workers here."""

    @property
    def device_sampling(self) -> bool:
        return self._pin_in is not None and not getattr(self.engine, "_parts", False) and os.environ.get("DL_HOST_SAMPLER") is None

    def prefill(self, tokens: Sequence[int], pos: int) -> None:
        """Evaluates tokens at positions pos..pos+n-1 without producing logits (prompt minus its last token)."""
        if tokens:
            self._send(OP_PREFILL, pos, tokens)
            self.engine.prefill(tokens, pos, want_logits=False)
            if self.draft is not None:
                self.draft.prefill(tokens, pos, want_logits=False)

    def forward_logits(self, token: int, pos: int) -> torch.Tensor:
        self._send(OP_STEP_LOGITS, pos, [token])
        return self.engine.step(token, pos)

    def decode_greedy(self, token: int, pos: int, n_steps: int) -> List[int]:
        """n greedy steps with the token fed back on the device (no host round trip per step): one control packet for all."""
        self._send(OP_DECODE_N, pos, [token, n_steps])
        return self.engine.decode_greedy(token, pos, n_steps)

    def forward_greedy(self, token: int, pos: int, logprobs: Optional[int] = None) -> int:
        """One step on the fused arg-max: H2D (token, pos) from pinned memory, forward, D2H of the token."""
        self._send(OP_STEP_GREEDY, pos, [token])
        eng = self.engine
        if self._pin_in is None:          # engine on the CPU (protocol tests)
            eng._set_inputs([token], pos)
            eng.run_decode_step()
            return int(eng.tokens[0])
        self._pin_in[0], self._pin_in[1] = token, pos
        eng.tokens[:1].copy_(self._pin_in[:1], non_blocking=True)
        eng.pos[:1].copy_(self._pin_in[1:2], non_blocking=True)
        eng.run_decode_step()
        return self._read_token(logprobs, controlled=False)

    def _read_token(self, logprobs: Optional[int], controlled: bool) -> int:
        """Enqueues the log-probabilities of the draw when asked, then copies the token back and waits for it."""
        eng = self.engine
        if logprobs is not None:
            eng.logprobs([logprobs], controlled=controlled)
        self._pin_out.copy_(eng.tokens[:1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        eng.check_abort()
        if logprobs is not None:
            self._last_logprobs = eng.read_logprobs()
        return int(self._pin_out[0])

    def next_token(self, token: int, pos: int, sampler, logprobs: Optional[int] = None) -> int:
        """One generated token at `pos` with the sampler's settings. Greedy with sampling controls runs on the device sampler
        (arg-max of the controlled logits), not on the fused arg-max. logprobs = k (0..20): also the log-probabilities of the
        drawn token and the k most likely ones, from the same logits the draw saw (last_logprobs()); the token is the same as
        without it."""
        if logprobs is not None:
            check_logprobs(logprobs, self.n_ranks)
        if sampler.temperature == 0.0 and not sampler.controls_active:
            return self.forward_greedy(token, pos, logprobs)
        if not self.device_sampling:
            t = int(sampler.sample(self.forward_logits(token, pos).float().cpu().numpy()))
            if logprobs is not None:
                self._last_logprobs = [self.engine.logprobs_host_draw(t, logprobs, sampler)]
            return t
        gen = (sampler.seed, sampler.seed_generation)
        if sampler.temperature != 0.0 and self._dev_seeded != gen:
            self.seed(sampler.seed)
            self._dev_seeded = gen
        key = sampler.completion_generation if sampler.controls_active else None
        if self._dev_controls != key:   # a new completion: count row 0 starts from zero
            self.set_controls(sampler, 1)
            self._dev_controls = key
        self.set_filters(sampler)
        self._send(OP_STEP_SAMPLE, pos, [token] + _f32_bits(sampler.temperature, sampler.topp))
        self.engine.step_sampled(token, pos, sampler.temperature, sampler.topp)
        return self._read_token(logprobs, controlled=True)

    def speculates(self, sampler) -> bool:
        """Whether a single completion with these sampler settings decodes in speculative rounds: a draft model is loaded and
        the draw is plain greedy (temperature 0, no penalties or logit bias). Requests with logprobs or n > 1 never do."""
        return self.draft is not None and sampler.temperature == 0.0 and not sampler.controls_active

    def spec_round(self, token: int, pos: int) -> List[int]:
        """One speculative round from the last emitted token at `pos` (runtime.engine.Engine.spec_round): the tokens greedy
        decoding emits next, one to draft_tokens + 1 of them."""
        toks, accepted, drafted = self.engine.spec_round(self.draft, token, pos, self.draft_tokens)
        self.spec_stats.add(drafted, accepted, len(toks))
        return toks

    def last_logprobs(self) -> list:
        """Per row of the last step that was asked for logprobs (next_token: one row; choices_first / choices_step: one per
        choice, None for inactive ones): (token id, logprob, [(id, logprob), ...] the k most likely in order of logprob desc,
        id asc). logprob(i) = x[i] - logsumexp(x) over the tokenizer's vocabulary, x the logits after logit_bias and the
        penalties (before temperature and top-p)."""
        return self._last_logprobs

    # ---- the device sampler's state, the same on every rank ----
    def seed(self, seed: int) -> None:
        """Seeds the single-sequence device generator."""
        self._send(OP_SEED, 0, _split_seed(seed))
        self.engine.seed_sampler(seed)

    def set_controls(self, sampler, row_mask: int) -> None:
        """The sampler's penalties and logit bias for the following draws; zeroes the count rows in row_mask."""
        bias = sampler.logit_bias
        words = _f32_bits(sampler.presence_penalty, sampler.frequency_penalty) + [row_mask]
        for t, v in bias:
            words += [t] + _f32_bits(v)
        self._send(OP_CONTROLS, 0, words)
        self.engine.set_sampling_controls(sampler.presence_penalty, sampler.frequency_penalty, bias, row_mask)

    def set_filters(self, sampler) -> None:
        """The sampler's top_k / min_p, before the first draw that uses them (under tensor parallelism each rank draws from
        the gathered logits with its own generator, so all ranks must hold the same filters)."""
        key = (sampler.top_k, sampler.min_p)
        if self._dev_filters != key:
            self._send(OP_FILTERS, 0, [key[0]] + _f32_bits(key[1]))
            self.engine.set_sampling_filters(*key)
            self._dev_filters = key

    # ---- several completions of one prompt (run_choices) ----
    def forget_device_seed(self):
        self._dev_seeded = None

    def save_sampler(self):
        key = self._dev_seeded
        return key, (self.engine.sampler_state() if key is not None and self.device_sampling else 0)

    def restore_sampler(self, saved):
        key, state = saved
        if key is not None and self.device_sampling:
            self.seed(state)
        self._dev_seeded = key

    def batched_choices(self, n: int) -> bool:
        return self.device_sampling and self.engine.supports_choices(n)

    def choice_controls(self, sampler, n: int) -> None:
        """The sampler's controls and filters for the batched choices, count rows 1..n zeroed."""
        self.set_filters(sampler)
        if sampler.controls_active or self._dev_controls is not None:
            self.set_controls(sampler, ((1 << n) - 1) << 1)
            self._dev_controls = -1 if sampler.controls_active else None   # row 0's counts are not this sampler's

    def seed_choices(self, seeds: Sequence[int]) -> None:
        self._send(OP_CHOICES_SEED, 0, [w for s in seeds for w in _split_seed(s)])
        self.engine.seed_choice_samplers(seeds)

    def choices_first(self, token: int, P: int, n: int, temperature: float, topp: float, logprobs: Optional[int] = None) -> List[int]:
        self._send(OP_CHOICES_FIRST, P, [token, n] + _f32_bits(temperature, topp))
        out = self.engine.choices_first(token, P, n, temperature, topp, **_lp_kw(logprobs))
        if logprobs is not None:
            self._last_logprobs = self.engine.read_logprobs()
        return out

    def choices_step(self, tokens: Sequence[int], P: int, C: int, j: int, active: Sequence[bool], temperature: float,
                     topp: float, logprobs: Optional[int] = None) -> List[int]:
        self._send(OP_CHOICES_STEP, P, [C, j, _active_mask(active)] + _f32_bits(temperature, topp) + list(tokens))
        out = self.engine.choices_step(tokens, P, C, j, active, temperature, topp, **_lp_kw(logprobs))
        if logprobs is not None:
            self._last_logprobs = self.engine.read_logprobs()
        return out


class ParallelRefused(ValueError):
    """A --parallel value this configuration cannot serve (see parallel_refusal)."""


def parallel_refusal(parallel: int, n_ranks: int = 1, n_experts: int = 0, cache: str = "split") -> Optional[str]:
    """Why `parallel` concurrent sequences (KV-cache slots) in layout `cache` cannot run in this configuration, or None if
    they can."""
    if cache not in SLOT_CACHE_LAYOUTS:
        return f"--parallel-cache must be split or paged, not {cache!r}"
    if not 1 <= parallel <= MAX_CHOICES:
        return f"--parallel must be from 1 to {MAX_CHOICES}"
    if parallel == 1:
        return None
    if n_ranks > 1:
        return "--parallel > 1 runs on one GPU only (workers cannot mirror slot steps yet)"
    if n_experts > 0:
        return "--parallel > 1 does not support mixture-of-experts models (the batched step has no MoE path)"
    if os.environ.get("DL_COLLECTIVES") == "nccl":
        return "--parallel > 1 does not support DL_COLLECTIVES=nccl"
    if os.environ.get("DL_HOST_SAMPLER") is not None:
        return "--parallel > 1 samples on the device: unset DL_HOST_SAMPLER"
    return None


class SlotRequest:
    """One request of a SlotScheduler. The server fills in the fields and overrides the hooks; the scheduler calls them on its
    engine thread.

    n: completions; temperature / topp / presence / frequency / bias / top_k / min_p: the sampling settings; seed: the
    request's seed or None; max_tokens (<= 0: no limit but the slot's context); logprobs: k (0..20) top entries of the
    log-probabilities of every token, passed to on_logprobs, or None."""
    n = 1
    temperature, topp, presence, frequency = 0.0, 0.9, 0.0, 0.0
    bias: Sequence = ()
    top_k, min_p = 0, 0.0
    seed: Optional[int] = None
    max_tokens = -1
    logprobs: Optional[int] = None

    def on_logprobs(self, i: int, entry: tuple) -> None:
        """With logprobs set: the entry (token, logprob, [(id, logprob), ...]) of completion i's next token, right before
        on_token is called with that token."""

    def cached_prefix(self, slot: int) -> int:
        """How many of the request's messages slot `slot`'s prompt cache covers (slot choice; ties go to the lowest index)."""
        return 0

    def prompt_len(self, slot: int) -> int:
        """P, the position of the prompt's last token, as prepare(slot) would return it, without changing anything (paged slots:
        what the request reserves before it is admitted)."""
        raise NotImplementedError

    def prepare(self, slot: int):
        """Resolves the prompt against slot `slot`'s cache: (tokens to prefill, their start position, last prompt token, P)
        with P = the last prompt token's position."""
        raise NotImplementedError

    def on_token(self, i: int, token: int) -> bool:
        """Token of completion i; True when completion i is finished (end of sequence or stop string)."""
        raise NotImplementedError

    def finish(self, out: List[List[int]], slots: List[int], P: int) -> None:
        """Every completion is done: out[i] holds completion i's tokens."""

    def fail(self, error: Exception, slots: List[int]) -> None:
        """The request ended early: refused (slots == []), or a client write, the prefill or the step failed. Its slots are
        already free; what they hold may no longer match what their prompt caches say."""


class SlotScheduler:
    """Serves SlotRequests on the KV-cache slots of a backend by the rules both API servers share (csrc/host/slot_scheduler.hpp):
    run() is the engine loop until stop(); submit and stop may be called from any thread; on_evict(slot) follows the eviction of a
    paged slot's idle cache. A hook's exception reaches the request's fail as it is, the scheduler's own refusals as ValueError.

    `backend` provides slots, slot_len, slot_prefill(slot, tokens, pos), slot_copy(src, dst, P),
    slot_sampling(slot, seed, temperature, topp, presence, frequency, bias, top_k=.., min_p=..) (the filters are passed only
    when one is on) and slots_step(tokens, pos, active) (InferenceSession(parallel=N)); for requests with logprobs also
    slot_logprobs(slot, k) and slots_step_logprobs(tokens, pos, active) -> (draws, per-slot entries), used only while such a
    request holds a slot. Paged backends (backend.paged true) also provide slot_reserve(slot, rows) -> bool,
    slot_trim(slot, rows), slot_release(slot), free_pages() and slot_pages(slot)."""

    def __init__(self, backend, seed_source: Callable[[], int], on_evict: Optional[Callable[[int], None]] = None):
        self._core = host().SlotScheduler(backend, seed_source, on_evict)

    def submit(self, req: SlotRequest) -> None:
        """Queues the request; one for no completions or for more completions than there are slots fails at once (no slots)."""
        self._core.submit(req)

    def stop(self) -> None:
        """run() returns before its next step."""
        self._core.stop()

    def run(self) -> None:
        """The engine loop, until stop(). While idle it still raises what a signal handler raises (Ctrl-C: KeyboardInterrupt)."""
        self._core.run()


class InferenceSession(TokenSteps):
    def __init__(self, model_path: str, tokenizer_path: Optional[str] = None, max_seq_len: int = 0,
                 temperature: float = 0.0, topp: float = 0.9, seed: int = 12345, device: Optional[str] = None,
                 max_batch: int = 8, use_pdl: bool = True, comm=None, moe_mode: str = "auto", presence_penalty: float = 0.0,
                 frequency_penalty: float = 0.0, logit_bias: Optional[dict] = None, parallel: int = 1,
                 kv_cache_float_type: str = "bf16", top_k: int = 0, min_p: float = 0.0, parallel_cache: str = "split",
                 draft_model: Optional[str] = None, draft_tokens: int = 3):
        """presence_penalty, frequency_penalty and logit_bias ({token id: value}) are the sampling controls of every
        completion (host Sampler.set_controls; they may be changed later through self.sampler.set_controls, which restarts the
        counts of the current completion). top_k and min_p are the sampling filters of every sampled draw (host
        Sampler.set_filters, 0: off; self.sampler.set_filters changes them). parallel > 1 splits the KV cache into that many slots for SlotScheduler
        (slot_prefill, slot_copy, slot_sampling, slots_step); the single-sequence calls then must not be used.
        kv_cache_float_type: "bf16" or "q80" (runtime.engine.Engine). parallel_cache: the layout of the slots, "split" (each
        slot owns floor(context / parallel) rows) or "paged" (the slots share the cache as one pool of 64-row pages, so one
        request may use the whole context; see SlotScheduler for the rules). draft_model: the `.m` file of a smaller model with the
        target's tokenizer; single greedy completions then decode in speculative rounds of draft_tokens (1, 3 or 7) drafts that
        this model checks in one batched forward, with the tokens of plain greedy decoding (DraftRefused where it cannot run)."""
        from .models.loader import load_device_weights
        from .runtime.engine import Engine

        self.model_file = ModelFile(model_path, max_seq_len)
        self.header = self.model_file.header
        self.comm = comm
        why = parallel_refusal(parallel, comm.world_size if comm is not None else 1, self.header.n_experts, parallel_cache)
        if why:
            raise ParallelRefused(why)
        rank = comm.rank if comm is not None else 0
        n_ranks = comm.world_size if comm is not None else 1
        draft_file = None
        if draft_model is not None:
            # the draft follows the target's context length and KV-cache storage
            draft_file = ModelFile(draft_model, self.header.seq_len)
            why = draft_refusal(draft_tokens, n_ranks, parallel, (("target model", self.header), ("draft model", draft_file.header)))
            if why:
                raise DraftRefused(why)
        if device is None:
            device = f"cuda:{torch.cuda.current_device()}"
        self.weights = load_device_weights(self.model_file, rank, n_ranks, torch.device(device), moe_mode=moe_mode, comm=comm)
        draft = None
        if draft_file is not None:
            draft = Engine(load_device_weights(draft_file, 0, 1, torch.device(device)), max_batch=max_batch, use_pdl=use_pdl,
                           kv_cache_float_type=kv_cache_float_type)
        super().__init__(Engine(self.weights, max_batch=max_batch, use_pdl=use_pdl, comm=comm, kv_cache_float_type=kv_cache_float_type),
                         device, n_ranks, draft, draft_tokens)
        H = host()
        self.tokenizer = H.Tokenizer(tokenizer_path) if tokenizer_path else None
        vocab = self.tokenizer.vocab_size if self.tokenizer else self.header.vocab_size
        self.sampler = H.Sampler(vocab, temperature, topp, seed)
        self.sampler.set_controls(presence_penalty, frequency_penalty, sorted((int(k), float(v)) for k, v in (logit_bias or {}).items()))
        self.sampler.set_filters(top_k, min_p)
        if self.tokenizer and self.tokenizer.vocab_size < self.header.vocab_size:
            for e in (self.engine, self.draft):
                if e is not None:
                    e.set_vocab_limit(self.tokenizer.vocab_size)
        self.pos = 0
        self.slots = parallel
        if parallel > 1:
            self.engine.set_slots(parallel, parallel_cache)
        self.slot_len = self.engine.slot_len
        self.paged = self.engine.paged

    # ---- KV-cache slots (SlotScheduler) ----
    def slot_prefill(self, slot: int, tokens: Sequence[int], pos: int) -> None:
        self.engine.slot_prefill(slot, tokens, pos)

    def slot_copy(self, src: int, dst: int, P: int) -> None:
        self.engine.slot_copy(src, dst, P)

    def slot_reserve(self, slot: int, rows: int) -> bool:
        return self.engine.slot_reserve(slot, rows)

    def slot_release(self, slot: int) -> None:
        self.engine.slot_release(slot)

    def slot_trim(self, slot: int, rows: int) -> None:
        self.engine.slot_trim(slot, rows)

    def free_pages(self) -> int:
        return self.engine.free_pages()

    def slot_pages(self, slot: int) -> List[int]:
        return self.engine.slot_pages(slot)

    def slot_sampling(self, slot: int, seed: int, temperature: float, topp: float, presence: float, frequency: float, bias, *,
                      top_k: int = 0, min_p: float = 0.0) -> None:
        self.engine.slot_sampling(slot, seed, temperature, topp, presence, frequency, bias, top_k=top_k, min_p=min_p)

    def slots_step(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]) -> List[int]:
        return self.engine.slots_step(tokens, pos, active)

    def slot_logprobs(self, slot: int, k: Optional[int]) -> None:
        self.engine.slot_logprobs(slot, k)

    def slots_step_logprobs(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]):
        return self.engine.slots_step_logprobs(tokens, pos, active)

    # ---- token level: the session's position by default, moved past what ran ----
    def reset(self):
        self.pos = 0

    def prefill(self, tokens: Sequence[int], pos: Optional[int] = None) -> None:
        pos = self.pos if pos is None else pos
        super().prefill(tokens, pos)
        self.pos = pos + len(tokens)

    def forward_logits(self, token: int, pos: Optional[int] = None) -> torch.Tensor:
        pos = self.pos if pos is None else pos
        lg = super().forward_logits(token, pos)
        self.pos = pos + 1
        return lg

    def next_token(self, token: int, pos: Optional[int] = None, sampler=None, logprobs: Optional[int] = None) -> int:
        """TokenSteps.next_token with the session's position and sampler by default; run_choices passes its own."""
        pos = self.pos if pos is None else pos
        tok = super().next_token(token, pos, self.sampler if sampler is None else sampler, logprobs)
        self.pos = pos + 1
        return tok

    def generate_choices(self, prompt: str, n: int, max_tokens: int, seed: Optional[int] = None, stop=None) -> List[str]:
        """n completions of `prompt`, each at most max_tokens tokens (and at most its share of the remaining context, see
        run_choices), with the session's temperature and top-p. Choice i is seeded with choice_seed(seed, i); without a seed
        the base seed is drawn from the session's sampler, so repeated calls differ. The prompt is prefilled once.
        stop: a string or a list of up to 4 strings (check_stop); each choice ends at the token that completes the first
        occurrence of any of them in its text, which is cut right before that occurrence (host StopMatcher)."""
        assert self.tokenizer is not None
        H = host()
        stops = check_stop(stop)
        toks = self.tokenizer.encode(prompt, True, True)
        self.prefill(toks[:-1])
        P = self.pos
        decoders = [H.TokenDecoder() for _ in range(n)]
        matchers = [H.StopMatcher(stops) for _ in range(n)] if stops else None
        pieces: List[List[bytes]] = [[] for _ in range(n)]

        def on_token(i: int, tok: int) -> bool:
            piece = decoders[i].decode(self.tokenizer, tok)
            if matchers:
                pieces[i].append(matchers[i].push(piece))
                if matchers[i].stopped:
                    return True
            else:
                pieces[i].append(piece)
            return bool(self.tokenizer.is_eos(tok))

        base = self.sampler.next_seed() if seed is None else seed
        run_choices(self, toks[-1], P, n, max_tokens, self.engine.seq_len, self.sampler, base, on_token)
        self.pos = P + 1
        if matchers:
            for i in range(n):
                pieces[i].append(matchers[i].flush())
        return [b"".join(p).decode("utf-8", errors="replace") for p in pieces]

    # ---- text level ----
    def generate(self, prompt: str, steps: int, on_piece: Optional[Callable[[str], None]] = None) -> str:
        assert self.tokenizer is not None
        toks = self.tokenizer.encode(prompt, True, True)
        self.prefill(toks[:-1])
        tok = toks[-1]
        self.tokenizer.reset_decoder()
        self.sampler.begin_completion()
        out = []
        limit = min(steps, self.header.seq_len)
        spec = self.speculates(self.sampler)
        while self.pos < limit:
            toks = self.spec_round(tok, self.pos) if spec else [super().next_token(tok, self.pos, self.sampler)]
            for tok in toks:
                self.pos += 1
                piece = self.tokenizer.decode(tok).decode("utf-8", errors="replace")
                out.append(piece)
                if on_piece:
                    on_piece(piece)
                if self.tokenizer.is_eos(tok):
                    return "".join(out)
                if self.pos >= limit:
                    break
        return "".join(out)
