"""Concurrent chat requests in the Python API server (`--parallel N`, api.SlotScheduler) on the CPU, over a stub slot backend
whose step takes a fixed time, so that requests really overlap."""
import http.client
import json
import os
import re
import socket
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest

from distributed_llama_b200 import host


class SlotStub:
    """N KV-cache slots: a row's next token depends on (token, position, its slot's seed when sampling), never on the slot index
    or on the other rows; its log-probability entry is a fixed float32 function of (drawn token, position, k). Every call is
    logged, and `log` keeps the prefills, copies and seeds as the native stub prints them."""

    def __init__(self, slots, slot_len, regular, eos, eos_after=10, delay=0.02):
        self.slots, self.slot_len, self.regular, self.eos, self.eos_after, self.delay = slots, slot_len, regular, eos, eos_after, delay
        self.seed, self.temp, self.produced, self.k = [0] * slots, [0.0] * slots, [0] * slots, [None] * slots
        self.prefills, self.copies, self.sampling, self.log = [], [], [], []
        self.max_active = 0

    def slot_prefill(self, slot, tokens, pos):
        self.prefills.append((slot, pos, len(tokens)))
        self.log.append(f"POS {slot} {pos} {len(tokens)}")

    def slot_copy(self, src, dst, P):
        self.copies.append((src, dst, P))
        self.log.append(f"COPY {src} {dst} {P}")

    def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias):
        self.sampling.append(slot)
        self.log.append(f"SEED {slot} {seed}")
        self.seed[slot], self.temp[slot], self.produced[slot], self.k[slot] = seed, temperature, 0, None

    def slot_logprobs(self, slot, k):
        self.k[slot] = k

    def slots_step_logprobs(self, tokens, pos, active):
        drawn = self.slots_step(tokens, pos, active)
        entries = []
        for b, t in enumerate(drawn):
            k = self.k[b] if active[b] else None
            entries.append(None if k is None else
                           (t, float(-np.float32(pos[b] % 7) * np.float32(0.37)),
                            [((t + 31 * j) % self.regular, float(-np.float32(j) * np.float32(0.2517) - np.float32(0.001))) for j in range(k)]))
        return drawn, entries

    def slots_step(self, tokens, pos, active):
        time.sleep(self.delay)
        self.max_active = max(self.max_active, sum(active))
        out = []
        for b in range(self.slots):
            if not active[b]:
                out.append(-1)
                continue
            self.produced[b] += 1
            salt = (self.seed[b] % 997) * 31 if self.temp[b] > 0 else 0
            out.append(self.eos if self.produced[b] > self.eos_after else (tokens[b] * 7 + pos[b] * 13 + 5 + salt) % self.regular)
        return out


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture
def server(tmp_path):
    """Starts a --parallel 4 server over SlotStub for max_requests connections: (port, stub, join)."""
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer

    def start(max_requests, parallel=4, eos_after=10, delay=0.02):
        H = host()
        path = str(tmp_path / "tok.t")
        write_synthetic_tokenizer(path, 512, style="llama3")
        tok = H.Tokenizer(path)
        stub = SlotStub(parallel, 1024 // parallel, tok.regular_vocab_size, list(tok.eos_ids)[0], eos_after, delay)
        port = _free_port()
        args = parse_args(["--model", "stub.m", "--tokenizer", path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0",
                           "--parallel", str(parallel)], False)
        ctx = SimpleNamespace(args=args, sess=None, inference=stub, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 77),
                              header=SimpleNamespace(seq_len=1024, vocab_size=tok.vocab_size))
        th = threading.Thread(target=py_api.serve, args=(ctx, max_requests + 1), daemon=True)   # + the readiness probe
        th.start()
        for _ in range(200):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
                break
            except OSError:
                time.sleep(0.02)
        return port, stub, lambda: th.join(timeout=30)
    return start


def _post(port, body, stamps=None):
    """Response content of choice 0 (streamed or not); `stamps` collects the arrival time of every streamed chunk."""
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=30)
    try:
        c.request("POST", "/v1/chat/completions", body=body if isinstance(body, str) else json.dumps(body),
                  headers={"Content-Type": "application/json"})
        r = c.getresponse()
        if "event-stream" not in r.getheader("Content-Type", ""):
            return [ch["message"]["content"] for ch in json.loads(r.read())["choices"]]
        text, parts = "", {}
        while True:
            line = r.fp.readline()
            if not line:
                break
            line = line.decode("utf-8", errors="replace").strip()
            if line.startswith("data: {"):
                if stamps is not None:
                    stamps.append(time.monotonic())
                for ch in json.loads(line[6:])["choices"]:
                    parts[ch["index"]] = parts.get(ch["index"], "") + (ch.get("delta") or {}).get("content", "")
            if line == "data: [DONE]":
                break
        return [parts[i] for i in sorted(parts)]
    finally:
        c.close()


def _msgs(i):
    return [{"role": "user", "content": f"client {i} says hello " * (i + 1)}]


def _concurrent(port, bodies, stagger=0.0):
    out, stamps = [None] * len(bodies), [[] for _ in bodies]

    def go(i):
        try:
            out[i] = _post(port, bodies[i], stamps[i])
        except (ConnectionError, http.client.HTTPException, OSError) as e:
            out[i] = e
    ths = []
    for i in range(len(bodies)):
        ths.append(threading.Thread(target=go, args=(i,)))
        ths[-1].start()
        time.sleep(stagger)
    for th in ths:
        th.join(timeout=30)
    return out, stamps


BODIES = [dict(messages=_msgs(0), stream=True), dict(messages=_msgs(1), stream=True, temperature=0.8, seed=11),
          dict(messages=_msgs(2), max_tokens=5), dict(messages=_msgs(3), temperature=0.9, seed=5, stream=True),
          dict(messages=_msgs(4), temperature=0.7, seed=3)]


def test_concurrent_requests_overlap_and_match_alone(server):
    port, stub, join = server(2 * len(BODIES))
    alone = [_post(port, b) for b in BODIES]
    together, stamps = _concurrent(port, BODIES, stagger=0.005)
    join()
    assert together == alone                                 # five requests on four slots: the fifth queued and completed
    assert stub.max_active == 4
    assert stamps[1][0] < stamps[0][-1]                      # B's first chunk arrived before A's last
    assert all(len(a[0]) > 0 for a in alone)


def test_disconnect_and_malformed_body_leave_the_others_alone(server):
    port, stub, join = server(2 * 3 + 2, eos_after=30, delay=0.03)
    bodies = BODIES[:3]
    alone = [_post(port, b) for b in bodies]

    def quitter():
        s = socket.create_connection(("127.0.0.1", port))
        body = json.dumps(dict(messages=_msgs(9), stream=True)).encode()
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nContent-Type: application/json\r\nContent-Length: " + str(len(body)).encode() +
                  b"\r\n\r\n" + body)
        s.recv(64)                                           # the stream started
        s.close()

    def malformed():
        s = socket.create_connection(("127.0.0.1", port))
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nContent-Length: 9\r\n\r\n{not json")
        assert s.recv(64) == b""                             # closed without a response
        s.close()
    side = [threading.Thread(target=quitter), threading.Thread(target=malformed)]
    for t in side:
        t.start()
    together, _ = _concurrent(port, bodies)
    for t in side:
        t.join(timeout=30)
    join()
    assert together == alone


def test_prefix_reuse_per_slot(server):
    port, stub, join = server(4)
    first, _ = _concurrent(port, [dict(messages=_msgs(0)), dict(messages=_msgs(1))])
    slots_turn1 = {s: pos for s, pos, _ in stub.prefills}
    assert len(slots_turn1) == 2 and all(p == 0 for p in slots_turn1.values())
    follow = [dict(messages=_msgs(i) + [{"role": "assistant", "content": first[i][0]}, {"role": "user", "content": "more"}]) for i in (1, 0)]
    _concurrent(port, follow)
    join()
    turn2 = stub.prefills[2:]
    assert len(turn2) == 2
    assert all(pos > 0 for _, pos, _ in turn2)              # each follow-up found its own slot's cache
    assert sorted(s for s, _, _ in turn2) == sorted(slots_turn1)


def test_choices_take_slots_and_too_many_are_refused(server):
    port, stub, join = server(3)
    got = _post(port, dict(messages=_msgs(0), n=2, temperature=0.8, seed=4))
    assert len(got) == 2 and got[0] != got[1]
    assert len(stub.copies) == 1 and len(set(stub.sampling)) == 2
    H = host()
    assert stub.seed[stub.sampling[0]] == H.choice_seed(4, 0) and stub.seed[stub.sampling[1]] == H.choice_seed(4, 1)
    with pytest.raises((ConnectionError, http.client.HTTPException, OSError)):
        _post(port, dict(messages=_msgs(0), n=5, temperature=0.8))
    greedy = _post(port, dict(messages=_msgs(1), n=3, temperature=0))
    join()
    assert len(greedy) == 3 and greedy[0] == greedy[1] == greedy[2]


@pytest.mark.parametrize("argv,env", [(["--parallel", "0"], {}), (["--parallel", "9"], {}), (["--parallel", "2", "--gpus", "2"], {}),
                                      (["--parallel", "2", "--workers", "10.0.0.2:9999"], {}),
                                      (["--parallel", "2"], {"DL_COLLECTIVES": "nccl"}), (["--parallel", "2"], {"DL_HOST_SAMPLER": "1"})])
def test_startup_refusals(argv, env, monkeypatch, capsys):
    from distributed_llama_b200.apps import api_server as py_api
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert py_api.main(["--model", "m.m", "--tokenizer", "t.t"] + argv) == 1
    err = capsys.readouterr().err.strip()
    assert "--parallel" in err and len(err.splitlines()) == 1


def test_mixture_of_experts_is_refused():
    from distributed_llama_b200.api import parallel_refusal
    assert "mixture-of-experts" in parallel_refusal(4, 1, 8)
    assert parallel_refusal(4, 1, 0) is None and parallel_refusal(1, 2, 8) is None
