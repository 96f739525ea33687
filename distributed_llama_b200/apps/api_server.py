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
from typing import Dict, List, Optional, Tuple

from .. import host
from ..api import (MAX_CHOICES, MAX_TOP_LOGPROBS, ParallelRefused, SlotRequest, SlotScheduler, check_logprobs, parallel_refusal,
                   run_choices)
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

    def complete(self, req: HttpRequest):
        """n completions of one prompt (api.run_choices; n = 1 without `n`): the prompt is prefilled once. After one completion
        the cache keeps its answer too; after several it keeps only the prompt messages, so a follow-up that quotes any one
        choice reuses the prompt."""
        ctx, H = self.ctx, self.H
        tok, inf, h, smp = ctx.tokenizer, ctx.inference, ctx.header, ctx.sampler
        body = req.json or {}
        n = parse_n(body)
        # server defaults: --presence-penalty / --frequency-penalty (argument objects that predate them mean 0)
        presence, frequency, bias = parse_controls(body, smp.vocab_size, getattr(ctx.args, "presence_penalty", 0.0),
                                                   getattr(ctx.args, "frequency_penalty", 0.0))
        lp_k = parse_logprobs(body, getattr(getattr(inf, "comm", None), "world_size", 1))
        smp.set_controls(presence, frequency, bias)
        messages = [(m["role"], m["content"]) for m in body["messages"]]
        stream = bool(body.get("stream", False))
        max_tokens = int(body.get("max_tokens", -1))
        smp.set_temperature(float(body.get("temperature", ctx.args.temperature)))
        smp.set_topp(float(body.get("top_p", ctx.args.topp)))
        if "seed" in body:
            smp.set_seed(int(body["seed"]))
        # several completions: choice i uses choice_seed(base, i); without a seed the base is drawn from the advancing generator
        base_seed = smp.seed if "seed" in body else (smp.next_seed() if n > 1 else 0)
        delta_prompt, start_pos = self.cache.resolve_delta_prompt(list(messages))
        content, public = self.gen.generate(delta_prompt, True)
        print(f"🔹{content.decode('utf-8', errors='replace')}🔸", end="")
        tokens = tok.encode(content, start_pos == 0, True)
        n_prompt = len(tokens)
        prompt_end = min(start_pos + n_prompt - 1, h.seq_len)
        for m in delta_prompt:
            self.cache.push(prompt_end, m)
        dets = [H.EosDetector(*self.detector_args) for _ in range(n)]
        decoders = [H.TokenDecoder() for _ in range(n)]
        p = public.decode("utf-8", errors="replace")
        buffers = [p] * n
        lps = LogprobsLog(tok, n) if lp_k is not None else None
        if stream:
            req.write_stream_start()
            if p:
                for i in range(n):
                    req.write_stream_chunk("data: " + chunk_json(p, False, i, lps.take(i) if lps else None) + "\r\n\r\n")
        n_pref = prompt_end - start_pos
        inf.prefill(tokens[:n_pref], start_pos)
        token = tokens[n_pref] if n_pref < len(tokens) else tokens[-1]

        def on_token(i: int, t: int) -> bool:
            piece = decoders[i].decode(tok, t)
            if n == 1 and piece:
                print(piece.decode("utf-8", errors="replace"), end="", flush=True)
            kind = dets[i].append(t, piece)
            if lps:
                lps.consumed(i, kind == H.EOS)
            if kind in (H.NOT_EOS, H.EOS):
                delta = dets[i].get_delta()
                if delta:
                    d = delta.decode("utf-8", errors="replace")
                    if stream:
                        req.write_stream_chunk("data: " + chunk_json(d, False, i, lps.take(i) if lps else None) + "\r\n\r\n")
                    buffers[i] += d
                dets[i].reset()
            return kind == H.EOS

        out = run_choices(inf, token, prompt_end, n, max_tokens, h.seq_len, smp, base_seed, on_token,
                          **({"logprobs": lp_k, "on_logprobs": lps.on_logprobs} if lps else {}))
        if n == 1:
            end = prompt_end + len(out[0])
            if end == h.seq_len:
                self.cache.clear()
            else:
                self.cache.push(end, ("assistant", buffers[0]))
        if stream:
            for i in range(n):
                write_stream_finish(req, i, lps)
            req.write_stream_chunk("data: [DONE]")
            req.write_stream_end()
        else:
            n_completion = sum(len(o) for o in out)
            req.write_json(json.dumps({
                "id": "cmpl-j0", "object": "chat.completion", "created": int(time.time()), "model": "Distributed Model",
                "usage": {"completion_tokens": n_completion, "prompt_tokens": n_prompt, "total_tokens": n_prompt + n_completion},
                "choices": [choice_json(i, b, lps) for i, b in enumerate(buffers)]}))
        print("🔶" if n == 1 else f"({n} choices)🔶")

    def slot_request(self, req: HttpRequest, caches: List[NaiveCache], n_slots: int) -> SlotRequest:
        """A validated chat completion for SlotScheduler (--parallel > 1): the same fields, limits and responses as complete(),
        with the prompt cache of the slot the scheduler picks. Raises ValueError / KeyError on a malformed body."""
        ctx, H = self.ctx, self.H
        tok, smp = ctx.tokenizer, ctx.sampler
        body = req.json or {}
        n = parse_n(body)
        if n > n_slots:
            raise ValueError(f"'n' must not exceed --parallel ({n_slots})")
        presence, frequency, bias = parse_controls(body, smp.vocab_size, getattr(ctx.args, "presence_penalty", 0.0),
                                                   getattr(ctx.args, "frequency_penalty", 0.0))
        messages = [(m["role"], m["content"]) for m in body["messages"]]
        stream = bool(body.get("stream", False))
        temperature = float(body.get("temperature", ctx.args.temperature))
        if temperature < 0:
            raise ValueError("'temperature' must not be negative")
        lp_k = parse_logprobs(body)   # --parallel > 1 runs on one GPU
        detector_args, gen = self.detector_args, self.gen

        class Chat(SlotRequest):
            def cached_prefix(self, slot):
                items = caches[slot].items
                ok = len(messages) > len(items) and all(items[i][1] == messages[i] for i in range(len(items)))
                return len(items) if ok else 0

            def prepare(self, slot):
                cache = caches[slot]
                delta, start = cache.resolve_delta_prompt(list(messages))
                content, public = gen.generate(delta, True)
                tokens = tok.encode(content, start == 0, True)
                self.n_prompt = len(tokens)
                P = min(start + len(tokens) - 1, slot_len)
                p = public.decode("utf-8", errors="replace")
                self.buffers = [p] * n
                lps = self.lps
                if stream:
                    req.write_stream_start()
                    if p:
                        for i in range(n):
                            req.write_stream_chunk("data: " + chunk_json(p, False, i, lps.take(i) if lps else None) + "\r\n\r\n")
                for m in delta:
                    cache.push(P, m)
                self.slot_cache = cache
                n_pref = P - start
                return tokens[:n_pref], start, (tokens[n_pref] if n_pref < len(tokens) else tokens[-1]), P

            def on_logprobs(self, i, entry):
                self.lps.on_logprobs(i, entry)

            def on_token(self, i, t):
                piece = self.decoders[i].decode(tok, t)
                kind = self.dets[i].append(t, piece)
                lps = self.lps
                if lps:
                    lps.consumed(i, kind == H.EOS)
                if kind in (H.NOT_EOS, H.EOS):
                    delta = self.dets[i].get_delta()
                    if delta:
                        d = delta.decode("utf-8", errors="replace")
                        if stream:
                            req.write_stream_chunk("data: " + chunk_json(d, False, i, lps.take(i) if lps else None) + "\r\n\r\n")
                        self.buffers[i] += d
                    self.dets[i].reset()
                return kind == H.EOS

            def finish(self, out, slots, P):
                if n == 1:
                    end = P + len(out[0])
                    if end == slot_len:
                        self.slot_cache.clear()
                    else:
                        self.slot_cache.push(end, ("assistant", self.buffers[0]))
                for s in slots[1:]:   # they hold a copy of the prompt rows
                    caches[s].items = list(caches[slots[0]].items)
                if stream:
                    for i in range(n):
                        write_stream_finish(req, i, self.lps)
                    req.write_stream_chunk("data: [DONE]")
                    req.write_stream_end()
                else:
                    n_completion = sum(len(o) for o in out)
                    req.write_json(json.dumps({
                        "id": "cmpl-j0", "object": "chat.completion", "created": int(time.time()), "model": "Distributed Model",
                        "usage": {"completion_tokens": n_completion, "prompt_tokens": self.n_prompt,
                                  "total_tokens": self.n_prompt + n_completion},
                        "choices": [choice_json(i, b, self.lps) for i, b in enumerate(self.buffers)]}))
                print(f"🔶 slot {slots[0]}" + (f" ({n} choices)" if n > 1 else ""), flush=True)
                self.done()

            def fail(self, error, slots):
                for s in slots:   # their rows may not match what their caches say (e.g. a prefill that never ran)
                    caches[s].clear()
                print(f"Socket error: {error}", flush=True)
                self.done()

        slot_len = self.slot_len
        r = Chat()
        r.n, r.temperature, r.topp = n, temperature, float(body.get("top_p", ctx.args.topp))
        r.presence, r.frequency, r.bias = presence, frequency, bias
        r.seed = int(body["seed"]) if "seed" in body else None
        r.max_tokens = int(body.get("max_tokens", -1))
        r.logprobs = lp_k
        r.lps = LogprobsLog(tok, n) if lp_k is not None else None
        r.dets = [H.EosDetector(*detector_args) for _ in range(n)]
        r.decoders = [H.TokenDecoder() for _ in range(n)]
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
    sched = SlotScheduler(backend, ctx.sampler.next_seed)
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
        [--chat-template {llama2|llama3|deepSeek3|chatml}] [--parallel <n>]
        --parallel <n>: decode up to n (1..8) chat requests together, each in its own KV-cache slot of
                        floor(context / n) tokens; single GPU and dense models only
"""


def main(argv=None) -> int:
    import os
    argv = list(sys.argv[1:] if argv is None else argv)
    args = parse_args(argv, False)
    if args.help:
        sys.stderr.write(USAGE)
        return 0
    why = parallel_refusal(args.parallel, max(args.gpus, 1, int(os.environ.get("WORLD_SIZE", "1"))) + len(args.workers))
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
        except ParallelRefused as e:   # found once the model header is read (mixture of experts)
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
