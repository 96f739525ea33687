"""`dllama-api`: OpenAI-style HTTP server (reference src/dllama-api.cpp:43-632, src/api-types.hpp).

Routes: POST /v1/chat/completions (JSON or SSE-chunked stream), GET /v1/models, OPTIONS * (CORS pre-flight), else 404.
Single request at a time over one global KV sequence, with the reference's NaiveCache prefix reuse: if the new message
history extends the cached one, generation restarts from the cached end position instead of 0.
Deliberate fixes over the reference (SURVEY A.2): request `temperature`/`top_p` are applied, `finish_reason` is "stop"
on non-stream responses.
"""
from __future__ import annotations

import json
import re
import socket
import sys
import threading
import time
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple

from .. import host
from ..api import (MAX_CHOICES, MAX_TOP_LOGPROBS, DraftRefused, ParallelRefused, SlotRequest, SlotScheduler, check_logprobs,
                   check_stop, draft_refusal, parallel_refusal, run_choices)
from .args import AppArgs, parse_args
from .cli import make_chat_tools
from .runtime import AppContext, run_inference_app


class NaiveCache:
    """(endPos, message) per chat turn; reuse only if *all* cached messages are an exact prefix of the new history."""

    def __init__(self):
        self.items: List[Tuple[int, Tuple[str, str]]] = []

    def push(self, end_pos: int, msg: Tuple[str, str]):
        self.items.append((end_pos, msg))

    def clear(self):
        self.items.clear()

    def resolve_delta_prompt(self, messages: List[Tuple[str, str]]) -> Tuple[List[Tuple[str, str]], int]:
        n = len(self.items)
        if n == 0:
            return messages, 0
        if len(messages) > n and all(self.items[i][1] == messages[i] for i in range(n)):
            start = self.items[n - 1][0]
            print(f"🐤 Found naive cache for {n} messages, pos={start}")
            return messages[n:], start
        self.clear()
        return messages, 0


class HttpRequest:
    def __init__(self, conn: socket.socket):
        self.conn = conn
        self.method = "UNKNOWN"
        self.path = ""
        self.headers: Dict[str, str] = {}
        self.body = b""
        self.json = None

    @staticmethod
    def read(conn: socket.socket) -> "HttpRequest":
        req = HttpRequest(conn)
        data = b""
        while b"\r\n\r\n" not in data and b"\n\n" not in data:
            chunk = conn.recv(65536)
            if not chunk:
                raise ConnectionError("Error while reading headers from socket")
            data += chunk
        sep = b"\r\n\r\n" if b"\r\n\r\n" in data else b"\n\n"
        head, rest = data.split(sep, 1)
        lines = head.decode("latin-1").splitlines()
        parts = lines[0].split()
        if len(parts) >= 2:
            req.method, req.path = parts[0].upper(), parts[1]
        for ln in lines[1:]:
            if ":" in ln:
                k, v = ln.split(":", 1)
                req.headers[k.strip().lower()] = v.strip()
        length = int(req.headers.get("content-length", "0") or 0)
        if len(rest) > length > 0:
            raise ValueError("Received more body data than Content-Length header said")
        while len(rest) < length:
            chunk = conn.recv(length - len(rest))
            if not chunk:
                raise ConnectionError("Error while reading body from socket")
            rest += chunk
        req.body = rest
        if rest:
            req.json = json.loads(rest.decode("utf-8"))
        return req

    def _send(self, data: bytes):
        self.conn.sendall(data)

    def write_cors(self):
        self._send(b"HTTP/1.1 204 No Content\r\nAccess-Control-Allow-Origin: *\r\nAccess-Control-Allow-Methods: GET, POST, PUT, DELETE\r\n"
                   b"Access-Control-Allow-Headers: Content-Type, Authorization\r\nConnection: close\r\n\r\n")

    def write_not_found(self):
        self._send(b"HTTP/1.1 404 Not Found\r\nConnection: close\r\nContent-Length: 9\r\n\r\nNot Found")

    def write_json(self, text: str):
        body = text.encode("utf-8")
        self._send(b"HTTP/1.1 200 OK\r\nAccess-Control-Allow-Origin: *\r\nContent-Type: application/json; charset=utf-8\r\n"
                   b"Connection: close\r\nContent-Length: " + str(len(body)).encode() + b"\r\n\r\n" + body)

    def write_stream_start(self):
        self._send(b"HTTP/1.1 200 OK\r\nAccess-Control-Allow-Origin: *\r\nContent-Type: text/event-stream; charset=utf-8\r\n"
                   b"Connection: close\r\nTransfer-Encoding: chunked\r\n\r\n")

    def write_stream_chunk(self, data: str):
        b = data.encode("utf-8")
        self._send(("%x" % len(b)).encode() + b"\r\n" + b + b"\r\n")

    def write_stream_end(self):
        self._send(b"0000\r\n\r\n")


def parse_n(body: dict) -> int:
    """The request's `n` (completions of one prompt): absent means 1; anything but an integer in 1..MAX_CHOICES is refused."""
    n = body.get("n", 1)
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= MAX_CHOICES:
        raise ValueError(f"'n' must be an integer from 1 to {MAX_CHOICES}")
    return n


MAX_PENALTY = 2.0           # |presence_penalty|, |frequency_penalty|
MAX_LOGIT_BIAS = 100.0       # |logit_bias value|
MAX_LOGIT_BIAS_ENTRIES = 100  # one tensor-parallel control packet carries them all (both runtimes)


def _number(v, lo: float, hi: float, what: str) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not lo <= v <= hi:
        raise ValueError(f"'{what}' must be a number from {lo:g} to {hi:g}")
    return float(v)


def parse_controls(body: dict, vocab: int, presence: float, frequency: float):
    """The request's sampling controls: (presence_penalty, frequency_penalty, logit_bias as (id, value) pairs sorted by id).
    Absent penalties take the server's defaults. Penalties are numbers in [-2, 2]; logit_bias is an object of at most 100
    entries whose keys are decimal token ids in [0, vocab) without leading zeros and whose values are numbers in [-100, 100].
    Anything else is refused."""
    if "presence_penalty" in body:
        presence = _number(body["presence_penalty"], -MAX_PENALTY, MAX_PENALTY, "presence_penalty")
    if "frequency_penalty" in body:
        frequency = _number(body["frequency_penalty"], -MAX_PENALTY, MAX_PENALTY, "frequency_penalty")
    bias = body.get("logit_bias", {})
    if not isinstance(bias, dict) or len(bias) > MAX_LOGIT_BIAS_ENTRIES:
        raise ValueError(f"'logit_bias' must be an object of at most {MAX_LOGIT_BIAS_ENTRIES} entries")
    pairs = []
    for k, v in bias.items():
        if not re.fullmatch(r"0|[1-9][0-9]{0,9}", k) or int(k) >= vocab:
            raise ValueError(f"'logit_bias' keys must be token ids from 0 to {vocab - 1}")
        pairs.append((int(k), _number(v, -MAX_LOGIT_BIAS, MAX_LOGIT_BIAS, "logit_bias")))
    return presence, frequency, sorted(pairs)


MAX_TOP_K = 2**31 - 1


def parse_filters(body: dict, top_k: int, min_p: float):
    """The request's sampling filters: (top_k, min_p). Absent fields take the server's defaults. top_k is an integer from 0 to
    2^31 - 1 (0: off; k >= the vocabulary keeps every token), min_p a number from 0 to 1 (0: off). Booleans, non-integer top_k
    and values out of range are refused."""
    if "top_k" in body:
        k = body["top_k"]
        if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k <= MAX_TOP_K:
            raise ValueError(f"'top_k' must be an integer from 0 to {MAX_TOP_K}")
        top_k = k
    if "min_p" in body:
        min_p = _number(body["min_p"], 0.0, 1.0, "min_p")
    return int(top_k), float(min_p)


def parse_logprobs(body: dict, n_ranks: int = 1) -> Optional[int]:
    """The request's log-probabilities: None without them, else the number of top entries. `logprobs` is a boolean (absent:
    false); `top_logprobs`, an integer from 0 to 20 (absent: 0), is allowed only with `logprobs: true`. Anything else is refused,
    as is `logprobs: true` under tensor parallelism."""
    on = body.get("logprobs", False)
    if not isinstance(on, bool):
        raise ValueError("'logprobs' must be a boolean")
    k = body.get("top_logprobs", 0)
    if "top_logprobs" in body and not on:
        raise ValueError("'top_logprobs' needs 'logprobs': true")
    if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k <= MAX_TOP_LOGPROBS:
        raise ValueError(f"'top_logprobs' must be an integer from 0 to {MAX_TOP_LOGPROBS}")
    if not on:
        return None
    check_logprobs(k, n_ranks)
    return k


def parse_stop(body: dict) -> List[bytes]:
    """The request's `stop` strings as UTF-8 bytes (api.check_stop): absent, null and [] mean none; a string or an array of at
    most 4 strings of 1 to 256 bytes each, without unpaired surrogates. Anything else is refused."""
    return check_stop(body.get("stop"))


def _number_field(body: dict, key: str, default):
    v = body.get(key, default)
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise ValueError(f"'{key}' must be a number")
    return v


def parse_chat(body, defaults, vocab: int, max_n: int, n_ranks: int) -> SimpleNamespace:
    """A chat completion request: messages as (role, content) pairs, n, stream, max_tokens, temperature, topp, seed (None
    without one), presence, frequency, bias (parse_controls), top_k, min_p (parse_filters), logprobs (parse_logprobs) and stop
    (parse_stop).
    `defaults` holds the server's --temperature, --topp, penalties and filters; n may not exceed max_n (the slot count under
    --parallel); n_ranks > 1 (tensor parallelism) refuses logprobs. A body that is not an object, `messages` that are not a list of {role, content} objects
    with string values, a number field that is not a number, a negative temperature or a malformed control raise ValueError;
    a body without `messages` raises KeyError."""
    if not isinstance(body, dict):
        raise ValueError("request body must be a JSON object")
    n = parse_n(body)
    if n > max_n:
        raise ValueError(f"'n' must not exceed --parallel ({max_n})")
    # server defaults: --presence-penalty / --frequency-penalty (argument objects that predate them mean 0)
    presence, frequency, bias = parse_controls(body, vocab, getattr(defaults, "presence_penalty", 0.0),
                                               getattr(defaults, "frequency_penalty", 0.0))
    top_k, min_p = parse_filters(body, getattr(defaults, "top_k", 0), getattr(defaults, "min_p", 0.0))
    logprobs = parse_logprobs(body, n_ranks)
    stop = parse_stop(body)
    messages = body["messages"]
    if not isinstance(messages, list) or not all(isinstance(m, dict) and isinstance(m.get("role"), str) and
                                                 isinstance(m.get("content"), str) for m in messages):
        raise ValueError("'messages' must be a list of {role, content} objects")
    temperature = float(_number_field(body, "temperature", defaults.temperature))
    if temperature < 0:
        raise ValueError("'temperature' must not be negative")
    return SimpleNamespace(messages=[(m["role"], m["content"]) for m in messages], n=n, stream=bool(body.get("stream", False)),
                           max_tokens=int(_number_field(body, "max_tokens", -1)), temperature=temperature,
                           topp=float(_number_field(body, "top_p", defaults.topp)),
                           seed=int(_number_field(body, "seed", 0)) if "seed" in body else None,
                           presence=presence, frequency=frequency, bias=bias, logprobs=logprobs, top_k=top_k, min_p=min_p, stop=stop)


def logprob_entry(tokenizer, entry) -> dict:
    """The response form of one token's log-probabilities (api.run_choices on_logprobs entry): `bytes` are the token's piece,
    `token` those bytes decoded as UTF-8 with replacement."""
    def one(t: int, lp: float) -> dict:
        b = tokenizer.piece(t)
        return {"token": b.decode("utf-8", errors="replace"), "logprob": lp, "bytes": list(b)}
    t, lp, top = entry
    e = one(t, lp)
    e["top_logprobs"] = [one(i, v) for i, v in top]
    return e


class LogprobsLog:
    """Entries of the tokens of n choices: all of them for the final JSON, and those not yet sent for the stream. The token that
    ends a choice by end of sequence gets none."""

    def __init__(self, tokenizer, n: int):
        self.tokenizer = tokenizer
        self.next: List[Optional[dict]] = [None] * n
        self.all: List[List[dict]] = [[] for _ in range(n)]
        self.pending: List[List[dict]] = [[] for _ in range(n)]

    def on_logprobs(self, i: int, entry) -> None:
        self.next[i] = logprob_entry(self.tokenizer, entry)

    def consumed(self, i: int, eos: bool) -> None:
        """Choice i's token (the last one given to on_logprobs) went through on_token; eos: it ended the choice."""
        if not eos:
            self.all[i].append(self.next[i])
            self.pending[i].append(self.next[i])
        self.next[i] = None

    def take(self, i: int) -> List[dict]:
        out, self.pending[i] = self.pending[i], []
        return out


def chunk_json(delta: Optional[str], stop: bool, index: int = 0, logprobs: Optional[List[dict]] = None) -> str:
    """One stream chunk; `logprobs` (a list, possibly empty) adds the entries of the tokens consumed since the last chunk."""
    choice = {"index": index, "finish_reason": "stop" if stop else ""}
    if not stop:
        choice["delta"] = {"role": "assistant", "content": delta}
        if logprobs is not None:
            choice["logprobs"] = {"content": logprobs}
    return json.dumps({"id": "cmpl-c0", "object": "chat.completion", "created": int(time.time()), "model": "Distributed Model",
                       "choices": [choice]})


def write_stream_finish(req: "HttpRequest", i: int, lps: Optional[LogprobsLog]) -> None:
    """Choice i's stop chunk, after one delta chunk with empty content for log-probability entries still unsent."""
    if lps and lps.pending[i]:
        req.write_stream_chunk("data: " + chunk_json("", False, i, lps.take(i)) + "\r\n\r\n")
    req.write_stream_chunk("data: " + chunk_json(None, True, i) + "\r\n\r\n")


def choice_json(i: int, content: str, lps: Optional[LogprobsLog]) -> dict:
    c = {"index": i, "message": {"role": "assistant", "content": content}, "finish_reason": "stop"}
    if lps:
        c["logprobs"] = {"content": lps.all[i]}
    return c


class ChatResponse:
    """The response to one chat request: its n choices' decoders, stop detectors, texts and log-probability entries, written as
    stream chunks or as one `cmpl-j0` JSON body. With `stop` strings each choice also has a host StopMatcher after its detector.
    echo: print the tokens' pieces to stdout."""

    def __init__(self, api: "ApiServer", req: HttpRequest, chat: SimpleNamespace, echo: bool = False):
        H, n = api.H, chat.n
        self.req, self.stream, self.n, self.tok, self.H, self.echo = req, chat.stream, n, api.ctx.tokenizer, H, echo
        self.dets = [H.EosDetector(*api.detector_args) for _ in range(n)]
        self.matchers = [H.StopMatcher(chat.stop) for _ in range(n)] if chat.stop else None
        self.decoders = [H.TokenDecoder() for _ in range(n)]
        self.lps = LogprobsLog(self.tok, n) if chat.logprobs is not None else None
        self.buffers = [""] * n

    def _chunk(self, i: int, text: str) -> None:
        self.req.write_stream_chunk("data: " + chunk_json(text, False, i, self.lps.take(i) if self.lps else None) + "\r\n\r\n")

    def start(self, public: str) -> None:
        """Every choice's text starts with the prompt's public part; a stream sends its head and that part."""
        self.buffers = [public] * self.n
        if self.stream:
            self.req.write_stream_start()
            if public:
                for i in range(self.n):
                    self._chunk(i, public)

    def on_logprobs(self, i: int, entry) -> None:
        self.lps.on_logprobs(i, entry)

    def on_token(self, i: int, t: int) -> bool:
        """Choice i's next token; True when it ended the choice (end of sequence or stop string)."""
        H = self.H
        piece = self.decoders[i].decode(self.tok, t)
        if self.echo and piece:
            print(piece.decode("utf-8", errors="replace"), end="", flush=True)
        kind = self.dets[i].append(t, piece)
        if self.lps:
            self.lps.consumed(i, kind == H.EOS)
        if kind in (H.NOT_EOS, H.EOS):
            delta = self.dets[i].get_delta()
            if self.matchers:
                delta = self.matchers[i].push(delta)
            if delta:
                d = delta.decode("utf-8", errors="replace")
                if self.stream:
                    self._chunk(i, d)
                self.buffers[i] += d
            self.dets[i].reset()
        return kind == H.EOS or self.stopped(i)

    def stopped(self, i: int) -> bool:
        """Choice i ended at a stop string."""
        return bool(self.matchers) and self.matchers[i].stopped

    def text(self, i: int) -> str:
        """Choice i's content so far, bytes held back by its matcher included."""
        if not self.matchers:
            return self.buffers[i]
        return self.buffers[i] + self.matchers[i].held.decode("utf-8", errors="replace")

    def finish(self, out: List[List[int]], n_prompt: int) -> None:
        """Every choice is done (out[i]: choice i's tokens): the stop chunks and [DONE], or the JSON body. Bytes a matcher still
        holds (a choice that ended another way) join the text, in one delta chunk before the stop chunk of a stream."""
        for i in range(self.n):
            rest = self.matchers[i].flush().decode("utf-8", errors="replace") if self.matchers else ""
            self.buffers[i] += rest
            if self.stream:
                if rest:
                    self._chunk(i, rest)
                write_stream_finish(self.req, i, self.lps)
        if self.stream:
            self.req.write_stream_chunk("data: [DONE]")
            self.req.write_stream_end()
        else:
            n_completion = sum(len(o) for o in out)
            self.req.write_json(json.dumps({
                "id": "cmpl-j0", "object": "chat.completion", "created": int(time.time()), "model": "Distributed Model",
                "usage": {"completion_tokens": n_completion, "prompt_tokens": n_prompt, "total_tokens": n_prompt + n_completion},
                "choices": [choice_json(i, b, self.lps) for i, b in enumerate(self.buffers)]}))


def remember_answer(cache: NaiveCache, P: int, out0: List[int], text: str, ctx_len: int) -> None:
    """After a single completion of the prompt ending at P the cache keeps its answer too, unless it filled the context."""
    end = P + len(out0)
    if end == ctx_len:
        cache.clear()
    else:
        cache.push(end, ("assistant", text))


class ApiServer:
    def __init__(self, ctx: AppContext):
        self.ctx = ctx
        self.cache = NaiveCache()
        self.gen, _ = make_chat_tools(ctx)
        self.H = host()
        eos_ids = list(ctx.tokenizer.eos_ids)
        stops = [ctx.tokenizer.piece(i) for i in eos_ids]
        pad = max((len(x) for x in stops), default=0)
        self.detector_args = (eos_ids, stops, pad, pad)

    def prepare_prompt(self, cache: NaiveCache, messages: List[Tuple[str, str]], ctx_len: int, echo: bool = False):
        """Resolves `messages` against `cache` and records the messages still to be evaluated in it: (tokens to prefill, their
        start position, the last prompt token, P = its position, the prompt's token count, the public prompt). echo: print
        the prompt to stdout."""
        delta, start = cache.resolve_delta_prompt(list(messages))
        content, public = self.gen.generate(delta, True)
        if echo:
            print(f"🔹{content.decode('utf-8', errors='replace')}🔸", end="")
        tokens = self.ctx.tokenizer.encode(content, start == 0, True)
        P = min(start + len(tokens) - 1, ctx_len)
        for m in delta:
            cache.push(P, m)
        n_pref = P - start
        return (tokens[:n_pref], start, tokens[n_pref] if n_pref < len(tokens) else tokens[-1], P, len(tokens),
                public.decode("utf-8", errors="replace"))

    def complete(self, req: HttpRequest):
        """n completions of one prompt (api.run_choices; n = 1 without `n`): the prompt is prefilled once. After one completion
        the cache keeps its answer too; after several, or after one cut at a stop string (its KV rows hold tokens past the cut),
        it keeps only the prompt messages, so a follow-up that quotes any one choice reuses the prompt. The request's sampling
        settings stay with the server's sampler."""
        ctx = self.ctx
        inf, smp, seq_len = ctx.inference, ctx.sampler, ctx.header.seq_len
        chat = parse_chat(req.json, ctx.args, smp.vocab_size, MAX_CHOICES, getattr(getattr(inf, "comm", None), "world_size", 1))
        smp.set_controls(chat.presence, chat.frequency, chat.bias)
        smp.set_filters(chat.top_k, chat.min_p)
        smp.set_temperature(chat.temperature)
        smp.set_topp(chat.topp)
        if chat.seed is not None:
            smp.set_seed(chat.seed)
        # several completions: choice i uses choice_seed(base, i); without a seed the base is drawn from the advancing generator
        base_seed = smp.seed if chat.seed is not None else (smp.next_seed() if chat.n > 1 else 0)
        prefill, start, token, P, n_prompt, public = self.prepare_prompt(self.cache, chat.messages, seq_len, echo=True)
        resp = ChatResponse(self, req, chat, echo=chat.n == 1)
        resp.start(public)
        inf.prefill(prefill, start)
        out = run_choices(inf, token, P, chat.n, chat.max_tokens, seq_len, smp, base_seed, resp.on_token,
                          **({"logprobs": chat.logprobs, "on_logprobs": resp.on_logprobs} if resp.lps else {}))
        if chat.n == 1 and not resp.stopped(0):
            remember_answer(self.cache, P, out[0], resp.text(0), seq_len)
        resp.finish(out, n_prompt)
        print("🔶" if chat.n == 1 else f"({chat.n} choices)🔶")

    def slot_request(self, req: HttpRequest, caches: List[NaiveCache], n_slots: int) -> SlotRequest:
        """A validated chat completion for SlotScheduler (--parallel > 1): the same fields, limits and responses as complete(),
        with the prompt cache of the slot the scheduler picks. Raises ValueError / KeyError on a malformed body."""
        chat = parse_chat(req.json, self.ctx.args, self.ctx.sampler.vocab_size, n_slots, 1)   # --parallel > 1 runs on one GPU
        resp = ChatResponse(self, req, chat)
        api, slot_len, messages = self, self.slot_len, chat.messages
        lens = {}   # prompt_len by (start position, cached messages)

        class Chat(SlotRequest):
            def cached_prefix(self, slot):
                items = caches[slot].items
                ok = len(messages) > len(items) and all(items[i][1] == messages[i] for i in range(len(items)))
                return len(items) if ok else 0

            def prompt_len(self, slot):
                n = self.cached_prefix(slot)
                start = caches[slot].items[n - 1][0] if n else 0
                if (start, n) not in lens:   # the head of a blocked queue asks again before every step
                    content, _ = api.gen.generate(messages[n:], True)
                    lens[(start, n)] = min(start + len(api.ctx.tokenizer.encode(content, start == 0, True)) - 1, slot_len)
                return lens[(start, n)]

            def prepare(self, slot):
                prefill, start, token, P, self.n_prompt, public = api.prepare_prompt(caches[slot], messages, slot_len)
                resp.start(public)
                return prefill, start, token, P

            on_logprobs, on_token = resp.on_logprobs, resp.on_token

            def finish(self, out, slots, P):
                if chat.n == 1 and not resp.stopped(0):
                    remember_answer(caches[slots[0]], P, out[0], resp.text(0), slot_len)
                for s in slots[1:]:   # they hold a copy of the prompt rows
                    caches[s].items = list(caches[slots[0]].items)
                resp.finish(out, self.n_prompt)
                print(f"🔶 slot {slots[0]}" + (f" ({chat.n} choices)" if chat.n > 1 else ""), flush=True)
                self.done()

            def fail(self, error, slots):
                for s in slots:   # their rows may not match what their caches say (e.g. a prefill that never ran)
                    caches[s].clear()
                print(f"Socket error: {error}", flush=True)
                self.done()

        r = Chat()
        vars(r).update(vars(chat))   # the SlotRequest fields: n, temperature, topp, seed, max_tokens, logprobs, the controls and filters
        r.done = lambda: None
        return r

    def models(self, req: HttpRequest):
        name = self.ctx.args.model.replace("\\", "/").split("/")[-1]
        req.write_json(json.dumps({"object": "list", "data": [{"id": name, "object": "model", "created": 0, "owned_by": "user"}]}))


def serve_parallel(ctx: AppContext, srv: socket.socket, api: ApiServer, n_slots: int, max_requests: int = 0) -> None:
    """--parallel > 1: every connection is read and validated on its own thread; chat completions go to a SlotScheduler whose
    engine thread (this one) decodes up to n_slots requests together. A malformed body closes its connection without a response."""
    backend = ctx.sess if ctx.sess is not None else ctx.inference
    api.slot_len = backend.slot_len
    caches = [NaiveCache() for _ in range(n_slots)]
    sched = SlotScheduler(backend, ctx.sampler.next_seed, on_evict=lambda s: caches[s].clear())
    pending = threading.Semaphore(0)   # one release per finished connection

    def handle(conn):
        keep = False
        try:
            req = HttpRequest.read(conn)
            print(f"🔷 {req.method} {req.path}", flush=True)
            if req.method == "OPTIONS":
                req.write_cors()
            elif req.method == "POST" and req.path == "/v1/chat/completions":
                r = api.slot_request(req, caches, n_slots)

                def done():
                    conn.close()
                    pending.release()
                r.done = done
                keep = True
                sched.submit(r)
            elif req.method == "GET" and req.path == "/v1/models":
                api.models(req)
            else:
                req.write_not_found()
        except (ConnectionError, BrokenPipeError, ValueError, KeyError, TypeError, json.JSONDecodeError) as e:
            print(f"Socket error: {e}", flush=True)
        finally:
            if not keep:
                conn.close()
                pending.release()

    def accept():
        served = 0
        while max_requests == 0 or served < max_requests:
            conn, _ = srv.accept()
            threading.Thread(target=handle, args=(conn,), daemon=True).start()
            served += 1
        for _ in range(served):
            pending.acquire()
        sched.stop()

    threading.Thread(target=accept, daemon=True).start()
    sched.run()
    srv.close()


def serve(ctx: AppContext, max_requests: int = 0) -> None:
    a = ctx.args
    srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
    srv.bind((a.host, a.port))
    srv.listen(8)
    api = ApiServer(ctx)
    if a.host in ("0.0.0.0", "127.0.0.1"):
        print(f"Server URL: http://localhost:{a.port}/v1/", flush=True)
    n_slots = getattr(a, "parallel", 1)
    if n_slots > 1:
        serve_parallel(ctx, srv, api, n_slots, max_requests)
        return
    served = 0
    while max_requests == 0 or served < max_requests:
        conn, _ = srv.accept()
        try:
            req = HttpRequest.read(conn)
            print(f"🔷 {req.method} {req.path}")
            if req.method == "OPTIONS":
                req.write_cors()
            elif req.method == "POST" and req.path == "/v1/chat/completions":
                api.complete(req)
            elif req.method == "GET" and req.path == "/v1/models":
                api.models(req)
            else:
                req.write_not_found()
        except (ConnectionError, BrokenPipeError, ValueError, KeyError, json.JSONDecodeError) as e:
            print(f"Socket error: {e}")
        finally:
            conn.close()
            served += 1
    srv.close()


USAGE = """Usage: dllama-api {--model <path>} {--tokenizer <path>} [--host <addr>] [--port <p>]
        [--buffer-float-type {f32|f16|q40|q80}] [--max-seq-len <max>] [--gpus <n>] [--workers <ip:port> ...]
        [--temperature <temp>] [--topp <t>] [--presence-penalty <p>] [--frequency-penalty <f>] [--seed <s>]
        [--top-k <k>] [--min-p <p>] [--chat-template {llama2|llama3|deepSeek3|chatml}] [--parallel <n>]
        [--parallel-cache {split|paged}] [--draft-model <path>] [--draft-tokens {1|3|7}]
        --parallel <n>: decode up to n (1..8) chat requests together, each in its own KV-cache slot of
                        floor(context / n) tokens; single GPU and dense models only
        --parallel-cache paged: the slots share the KV cache as one pool of 64-token pages instead, so a request
                        may use the whole context while the pool has room (default split)
        --draft-model <path>: greedy single-completion requests decode in speculative rounds: the draft (same
                        tokenizer, dense q40) proposes --draft-tokens tokens (default 3), the model checks them at once
"""


def main(argv=None) -> int:
    import os
    argv = list(sys.argv[1:] if argv is None else argv)
    args = parse_args(argv, False)
    if args.help:
        sys.stderr.write(USAGE)
        return 0
    n_ranks = max(args.gpus, 1, int(os.environ.get("WORLD_SIZE", "1"))) + len(args.workers)
    why = parallel_refusal(args.parallel, n_ranks, 0, args.parallel_cache)
    if not why and args.draft_model is not None:
        why = draft_refusal(args.draft_tokens, n_ranks, args.parallel)
    if why:
        sys.stderr.write(why + "\n")
        return 1
    if args.gpus > 1 and os.environ.get("DLLAMA_SPAWNED") != "1" and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        # Supervisor of a tensor-parallel serving job: a rank that loses a peer (control-channel heartbeat, device-side wait timeout)
        # exits non-zero and torchrun tears the job down; the whole job is then started again after 3 s — the reference's root retry
        # loop + worker re-listen loop (dllama-api.cpp:616-628, app.cpp:306-365).
        import subprocess
        attempt = 0
        while True:
            port = 29500 + ((os.getpid() + 7 * attempt) % 2000)
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={args.gpus}", "--master-addr", "127.0.0.1",
                   "--master-port", str(port), "-m", "distributed_llama_b200.apps.api_server"] + argv
            try:
                rc = subprocess.call(cmd, env=dict(os.environ, DLLAMA_SPAWNED="1"))
            except KeyboardInterrupt:
                return 130
            if rc == 0 or rc < 0 or rc == 130:
                return rc
            print(f"🚨 Inference error: the tensor-parallel job exited with code {rc}\n🔄 Retrying in 3 seconds...", flush=True)
            time.sleep(3)
            attempt += 1
    # the reference retries runInferenceApp forever on connection / executor errors (dllama-api.cpp:616-628)
    while True:
        try:
            run_inference_app(args, serve)
            return 0
        except (ParallelRefused, DraftRefused) as e:   # found once the model headers are read
            sys.stderr.write(f"{e}\n")
            return 1
        except (ConnectionError, RuntimeError) as e:
            print(f"🚨 Inference error: {e}")
            if int(os.environ.get("WORLD_SIZE", "1")) > 1:
                return 1          # a lost rank cannot be re-joined from inside the job: the supervisor above restarts the whole job
            print("🔄 Retrying in 3 seconds...")
            time.sleep(3)
            args.info = False


if __name__ == "__main__":
    sys.exit(main())
