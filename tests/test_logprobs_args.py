"""`logprobs` / `top_logprobs` of the Python chat server without a GPU: parsing and refusals, the tensor-parallel refusal, entry
construction from token pieces, stream chunking of pending entries, and run_choices / SlotScheduler delivering entries."""
import json
import os
import re
import subprocess
import threading
from types import SimpleNamespace

import pytest

from distributed_llama_b200.api import SlotRequest, SlotScheduler, check_logprobs, run_choices
import test_sampling_controls as tsc  # its raw-socket client and parsed-response helpers
from distributed_llama_b200.apps.api_server import LogprobsLog, chunk_json, logprob_entry, parse_logprobs, write_stream_finish

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("body,want", [({}, None), ({"logprobs": False}, None), ({"logprobs": True}, 0),
                                       ({"logprobs": True, "top_logprobs": 0}, 0), ({"logprobs": True, "top_logprobs": 20}, 20)])
def test_parse_accepts(body, want):
    assert parse_logprobs(body) == want


@pytest.mark.parametrize("body", [{"logprobs": 1}, {"logprobs": "true"}, {"logprobs": None}, {"logprobs": True, "top_logprobs": 21},
                                  {"logprobs": True, "top_logprobs": -1}, {"logprobs": True, "top_logprobs": 1.0},
                                  {"logprobs": True, "top_logprobs": True}, {"top_logprobs": 2}, {"logprobs": False, "top_logprobs": 0}])
def test_parse_refuses(body):
    with pytest.raises(ValueError):
        parse_logprobs(body)


def test_tensor_parallel_refusal():
    with pytest.raises(ValueError, match="tensor parallelism"):
        parse_logprobs({"logprobs": True}, n_ranks=2)
    assert parse_logprobs({}, n_ranks=2) is None        # without the field tensor-parallel jobs serve as before
    with pytest.raises(ValueError):
        check_logprobs(3, 4)


class Tok:
    pieces = {0: b"a", 1: b"\xe2", 2: b"\x82\xac", 3: "€".encode(), 4: b"<|eot_id|>"}

    def piece(self, i):
        return self.pieces[i]


def test_entry_bytes_and_tokens():
    e = logprob_entry(Tok(), (1, -0.5, [(3, -0.25), (1, -0.5), (2, -3.0)]))
    assert e == {"token": "�", "logprob": -0.5, "bytes": [0xE2],
                 "top_logprobs": [{"token": "€", "logprob": -0.25, "bytes": [0xE2, 0x82, 0xAC]},
                                  {"token": "�", "logprob": -0.5, "bytes": [0xE2]},
                                  {"token": "��", "logprob": -3.0, "bytes": [0x82, 0xAC]}]}


class Req:
    def __init__(self):
        self.chunks = []

    def write_stream_chunk(self, data):
        self.chunks.append(json.loads(data[len("data: "):]) if data.startswith("data: {") else data)


def test_stream_chunking_of_pending_entries():
    log = LogprobsLog(Tok(), 2)
    req = Req()
    log.on_logprobs(0, (0, -1.0, []))
    log.consumed(0, eos=False)
    req.write_stream_chunk("data: " + chunk_json("a", False, 0, log.take(0)))
    log.on_logprobs(0, (1, -2.0, []))                  # held back: no text yet
    log.consumed(0, eos=False)
    log.on_logprobs(0, (4, -0.1, []))                  # end of sequence: no entry
    log.consumed(0, eos=True)
    log.on_logprobs(1, (3, -0.3, []))
    log.consumed(1, eos=False)
    write_stream_finish(req, 0, log)
    write_stream_finish(req, 1, log)
    c = [ch["choices"][0] for ch in req.chunks]
    assert [e["token"] for e in c[0]["logprobs"]["content"]] == ["a"]
    assert c[1]["delta"]["content"] == "" and [e["bytes"] for e in c[1]["logprobs"]["content"]] == [[0xE2]]
    assert c[2]["finish_reason"] == "stop" and "logprobs" not in c[2]
    assert c[3]["index"] == 1 and [e["token"] for e in c[3]["logprobs"]["content"]] == ["€"]
    assert c[4]["finish_reason"] == "stop"
    assert [len(x) for x in log.all] == [2, 1]
    assert "logprobs" not in json.loads(chunk_json("x", False, 0))["choices"][0]


class Smp:
    temperature, topp, vocab_size = 0.0, 0.9, 10
    presence_penalty = frequency_penalty = 0.0
    logit_bias = ()

    def begin_completion(self):
        pass


class Backend:
    """Greedy single sequence: token t + 1 each step, entries made up from the step."""

    def __init__(self):
        self.calls = []

    def next_token(self, token, pos, sampler, logprobs=None):
        self.calls.append(logprobs)
        self.last = [(token + 1, -float(pos), [(token + 1, -float(pos))] * (logprobs or 0))]
        return token + 1

    def last_logprobs(self):
        return self.last


def test_run_choices_delivers_entries_before_tokens():
    be = Backend()
    events = []
    out = run_choices(be, 5, 3, 2, 4, 100, Smp(), 0, lambda i, t: events.append(("tok", i, t)) or False, logprobs=1,
                      on_logprobs=lambda i, e: events.append(("lp", i, e[0])))
    assert out == [[6, 7, 8, 9]] * 2
    assert events[:4] == [("lp", 0, 6), ("tok", 0, 6), ("lp", 1, 6), ("tok", 1, 6)]   # greedy n: one list for every choice
    assert be.calls == [1] * 4
    be2 = Backend()
    run_choices(be2, 5, 3, 1, 2, 100, Smp(), 0, lambda i, t: False)
    assert be2.calls == [None, None]                   # without logprobs the backend is called as before


class SlotBackend:
    slots, slot_len = 2, 64

    def __init__(self):
        self.lp = {}

    def slot_prefill(self, slot, tokens, pos):
        pass

    def slot_copy(self, src, dst, P):
        pass

    def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias):
        self.lp.pop(slot, None)

    def slot_logprobs(self, slot, k):
        self.lp[slot] = k

    def slots_step(self, tokens, pos, active):
        return [t + 1 for t in tokens]

    def slots_step_logprobs(self, tokens, pos, active):
        return self.slots_step(tokens, pos, active), [((t + 1, -1.0, []) if a and s in self.lp else None)
                                                      for s, (t, a) in enumerate(zip(tokens, active))]


def test_slot_scheduler_delivers_entries():
    got = {}

    class R(SlotRequest):
        def __init__(self, name, k):
            self.name, self.logprobs, self.max_tokens = name, k, 3
            got[name] = []

        def prepare(self, slot):
            return [], 0, 10, 0

        def on_logprobs(self, i, entry):
            got[self.name].append(("lp", entry[0]))

        def on_token(self, i, t):
            got[self.name].append(("tok", t))
            return False

        def finish(self, out, slots, P):
            done.release()

    done = threading.Semaphore(0)
    be = SlotBackend()
    sched = SlotScheduler(be, lambda: 1)
    th = threading.Thread(target=sched.run)
    th.start()
    sched.submit(R("a", 2))
    sched.submit(R("b", None))
    assert done.acquire(timeout=10) and done.acquire(timeout=10)
    sched.stop()
    th.join(timeout=10)
    assert got["a"] == [("lp", 11), ("tok", 11), ("lp", 12), ("tok", 12), ("lp", 13), ("tok", 13)]
    assert got["b"] == [("tok", 11), ("tok", 12), ("tok", 13)]


# ---- both servers over a stub model ----------------------------------------------------------------------------------------------

class LogprobsStub:
    """tests/native/api_logprobs_stub_main.cpp in Python."""

    def __init__(self, V, eos, tp=False):
        import numpy as np
        self.np, self.V, self.eos, self.end, self.k, self.last = np, V, eos, 0, None, None
        self.comm = SimpleNamespace(world_size=2) if tp else None
        self.t_hash = (np.arange(V, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)

    def prefill(self, tokens, pos):
        self.end = pos + len(tokens)

    def next_token(self, token, pos, sampler, logprobs=None):
        np = self.np
        t = self.eos
        if pos + 1 - self.end <= 12:
            k = ((self.t_hash[:sampler.vocab_size] + np.uint64(token * 97 + pos * 13)) & np.uint64(0xFFFFFFFF)) % np.uint64(1000)
            t = int(sampler.sample(k.astype(np.float32) / np.float32(100.0)))
        if logprobs is not None:
            lp = float(-np.float32(pos % 7) * np.float32(0.37))
            top = [((t + 31 * j) % self.V, float(-np.float32(j) * np.float32(0.2517) - np.float32(0.001))) for j in range(logprobs)]
            self.last = [(t, lp, top)]
        return t

    def last_logprobs(self):
        return self.last

    def forget_device_seed(self):
        pass

    def save_sampler(self):
        return None

    def restore_sampler(self, saved):
        pass

    def batched_choices(self, n):
        return False


@pytest.fixture(scope="module")
def lp_stub(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("api_logprobs"))
    exe = os.path.join(d, "api_logprobs_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_logprobs_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


def _lp_python(tok_path, bodies, tp=False):
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    H = host()
    tok = H.Tokenizer(tok_path)
    model = LogprobsStub(tok.vocab_size, list(tok.eos_ids)[0], tp)
    port = tsc._free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                          header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, len(bodies) + 1), daemon=True)
    th.start()
    tsc._wait(port)
    out = [tsc._post(port, b) for b in bodies]
    th.join(timeout=20)
    return out


def _lp_native(stub, bodies, tp=False):
    exe, tok_path = stub
    port = tsc._free_port()
    proc = subprocess.Popen([exe, tok_path, str(port), str(len(bodies) + 1)] + (["tp"] if tp else []), stdout=subprocess.PIPE,
                            stderr=subprocess.STDOUT, text=True)
    try:
        tsc._wait(port)
        return [tsc._post(port, b) for b in bodies]
    finally:
        try:
            proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.communicate()


MSGS = [{"role": "user", "content": "hello"}]
LP_BODIES = [dict(messages=MSGS, logprobs=True, top_logprobs=3), dict(messages=MSGS, logprobs=True, top_logprobs=2, stream=True),
             dict(messages=MSGS, logprobs=True, top_logprobs=20, n=3, temperature=0.8, seed=5),
             dict(messages=MSGS, logprobs=True, n=3, temperature=0.8, seed=5, stream=True, max_tokens=5),
             dict(messages=MSGS, logprobs=True, top_logprobs=1, max_tokens=4), dict(messages=MSGS, n=3, temperature=0.8, seed=5)]
BAD = [dict(messages=MSGS, logprobs=1), dict(messages=MSGS, logprobs=True, top_logprobs=21), dict(messages=MSGS, logprobs=True, top_logprobs=-1),
       dict(messages=MSGS, logprobs=True, top_logprobs=1.0), dict(messages=MSGS, logprobs=True, top_logprobs=True),
       dict(messages=MSGS, top_logprobs=2), dict(messages=MSGS, logprobs=None)]


def test_servers_agree_on_logprobs(lp_stub):
    py, nat = _lp_python(lp_stub[1], LP_BODIES), _lp_native(lp_stub, LP_BODIES)
    for i, (a, b) in enumerate(zip(py, nat)):
        assert a and tsc._parts(a) == tsc._parts(b), i
        # the logprobs are formatted alike, byte for byte (Python float repr, \\u escapes)
        assert re.findall(r'"logprob": [^,}]+', a) == re.findall(r'"logprob": [^,}]+', b), i
    j = json.loads(py[0])
    e = j["choices"][0]["logprobs"]["content"]
    assert e and all(len(x["top_logprobs"]) == 3 for x in e)
    assert "logprobs" not in py[5]
    # the stream's entries, concatenated, are the non-stream list; the last token before end of sequence has its entry
    stream = tsc._parts(py[1])
    assert sum(len(c["choices"][0].get("logprobs", {}).get("content", [])) for c in stream if isinstance(c, dict)) == 12


@pytest.mark.parametrize("server", ["python", "native"])
def test_malformed_logprobs_are_refused(lp_stub, server):
    ok = dict(messages=MSGS, logprobs=True, max_tokens=2)
    bodies = [x for b in BAD for x in (b, ok)]
    out = _lp_python(lp_stub[1], bodies) if server == "python" else _lp_native(lp_stub, bodies)
    for i in range(0, len(bodies), 2):
        assert out[i] == "", bodies[i]
        assert json.loads(out[i + 1])["choices"][0]["logprobs"]["content"][0]["top_logprobs"] == []


@pytest.mark.parametrize("server", ["python", "native"])
def test_tensor_parallel_refuses_logprobs_in_both_servers(lp_stub, server):
    bodies = [dict(messages=MSGS, logprobs=True), dict(messages=MSGS, max_tokens=2)]
    out = _lp_python(lp_stub[1], bodies, tp=True) if server == "python" else _lp_native(lp_stub, bodies, tp=True)
    assert out[0] == "" and json.loads(out[1])["usage"]["completion_tokens"] == 2
