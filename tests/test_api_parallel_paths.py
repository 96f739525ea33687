"""Both API servers answer `--parallel` chat completions byte for byte as recorded. A fixed request matrix, sent one request after
another to a --parallel 4 server over the stub slot backends (tests/native/api_parallel_stub_main.cpp, and SlotStub in
tests/test_api_parallel.py, its twin in Python), was recorded before the single-sequence and slot paths of each server shared
their request code. Both servers must still give every response, apart from `created`, and make the same prefills, prompt copies
and slot seeds ("POS <slot> <start> <n>", "COPY <src> <dst> <P>", "SEED <slot> <seed>").

Re-record with `PYTHONPATH=. python tests/test_api_parallel_paths.py`: it runs the matrix against the Python server in this tree
and against the native stub, and keeps the native answer and lines of any cell where the two servers disagree under
"native_response" and "native_log".

The refusal tests send malformed bodies, each followed by a good request, to both request paths of both servers."""
import json
import os
import re
import subprocess
import tempfile
import threading
from types import SimpleNamespace

import pytest

from test_api_completion_paths import StubModel, _free_port, _post, _wait
from test_api_parallel import SlotStub
import test_sampling_controls as tsc  # its raw-socket client: "" when the server closed the connection without answering

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "api_parallel_completions.json")
PARALLEL, SLOT_LEN = 4, 256   # both stubs split 1024 rows over the slots
MSGS = [{"role": "system", "content": "be brief"}, {"role": "user", "content": "hello there"}]
LOG_LINE = re.compile(r"^(?:POS|COPY|SEED)(?: \d+)+$", re.M)


def _build_stub(d):
    exe = os.path.join(d, "api_parallel_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_parallel_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe, "-lpthread"], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


def _python_server(tok_path, n_requests, parallel, seq_len=1024):
    """A Python server for n_requests requests over SlotStub (parallel > 1) or StubModel: (port, model, join)."""
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    H = host()
    tok = H.Tokenizer(tok_path)
    eos = list(tok.eos_ids)[0]
    model = SlotStub(parallel, 1024 // parallel, tok.regular_vocab_size, eos, 10, 0.0) if parallel > 1 else StubModel(tok.regular_vocab_size, eos)
    port = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0",
                       "--parallel", str(parallel)], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 77),
                          header=SimpleNamespace(seq_len=seq_len, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, n_requests + 1), daemon=True)   # + the readiness probe
    th.start()
    _wait(port)
    return port, model, lambda: th.join(timeout=30)


def _run_python(tok_path, bodies):
    """Serves `bodies` one after another on a --parallel 4 Python server: (responses, each request's stub log lines)."""
    port, model, join = _python_server(tok_path, len(bodies), PARALLEL)
    out, logs = [], []
    for b in bodies:
        seen = len(model.log)
        out.append(_post(port, b(out) if callable(b) else b))
        logs.append(model.log[seen:])
    join()
    return out, logs


def _native_server(stub, n_requests, args=()):
    exe, tok_path = stub
    port = _free_port()
    proc = subprocess.Popen([exe, tok_path, str(port), str(n_requests + 1), *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    _wait(port)

    def log():
        try:
            return proc.communicate(timeout=30)[0]
        except subprocess.TimeoutExpired:
            proc.kill()
            return proc.communicate()[0]
    return port, log


def _run_native(stub, bodies):
    port, log = _native_server(stub, len(bodies), [str(PARALLEL), "10", "0"])
    try:
        out = [_post(port, b) for b in bodies]
    finally:
        text = log()
    # every request's lines follow the line its reader prints when it arrives
    per = [LOG_LINE.findall(part) for part in text.split("🔷 POST /v1/chat/completions")[1:]]
    return out, per


def _follow_up(messages, answer: int, choice: int, **extra):
    """A history that quotes choice `choice` of response `answer` of the same session."""
    def body(prev):
        j = json.loads(prev[answer])
        msgs = messages + [{"role": "assistant", "content": j["choices"][choice]["message"]["content"]}, {"role": "user", "content": "more"}]
        return dict(extra, messages=msgs)
    return body


def _long_messages(tok_path, P):
    """One user message whose prompt's last token sits at position P."""
    from distributed_llama_b200 import host
    H = host()
    tok = H.Tokenizer(tok_path)
    gen = H.ChatTemplateGenerator(H.TEMPLATE_UNKNOWN, tok.chat_template, tok.piece(list(tok.eos_ids)[0]))
    for k in range(1, 2 * SLOT_LEN):
        content, _ = gen.generate([("user", "a" * k)], True)
        if len(tok.encode(content, True, True)) - 1 == P:
            return [{"role": "user", "content": "a" * k}]
    raise AssertionError(f"no prompt ends at {P}")


def _matrix(tok_path):
    """(session name, cells): each cell is (name, body or body-builder over the earlier responses by index)."""
    def cell(**kw):
        return dict(kw, messages=MSGS)
    other = [{"role": "user", "content": "tell me more"}]
    main = [
        ("n-absent-t0", cell()),
        ("n-absent-t0-stream-max4", cell(stream=True, max_tokens=4)),
        ("n1-t0.8-seed", cell(n=1, temperature=0.8, seed=42)),
        ("n-absent-t0.8-noseed-stream-max6", cell(temperature=0.8, stream=True, max_tokens=6)),
        ("n2-t0.8-seed-stream", cell(n=2, temperature=0.8, seed=7, stream=True)),
        ("n4-t0.8-noseed-max4", cell(n=4, temperature=0.8, max_tokens=4)),
        ("n3-t0", cell(n=3, temperature=0)),
        ("n2-t0-stream-max4", cell(n=2, temperature=0, stream=True, max_tokens=4)),
        ("lp-k0", cell(logprobs=True)),
        ("lp-k3-stream-max5", cell(logprobs=True, top_logprobs=3, stream=True, max_tokens=5)),
        ("lp-k20-n2-t0.8-seed-max3", cell(logprobs=True, top_logprobs=20, n=2, temperature=0.8, seed=5, max_tokens=3)),
        ("lp-k3-n3-t0.8-seed-stream-max5", cell(logprobs=True, top_logprobs=3, n=3, temperature=0.8, seed=5, stream=True, max_tokens=5)),
        ("lp-k0-n3-t0-stream", cell(logprobs=True, top_logprobs=0, n=3, temperature=0, stream=True)),
        ("lp-k20-t0.8-noseed", cell(logprobs=True, top_logprobs=20, temperature=0.8, max_tokens=3)),
        ("controls-t0.8-seed", cell(temperature=0.8, seed=3, presence_penalty=1.5, frequency_penalty=-0.5, logit_bias={"5": -100, "300": 3.25})),
        ("controls-n2-t0.9-seed-stream", cell(n=2, temperature=0.9, top_p=0.5, seed=11, frequency_penalty=2, stream=True)),
        ("answer-n1", dict(messages=other, temperature=0.8, seed=3, max_tokens=6)),
        ("follow-up-after-n1", _follow_up(other, 16, 0, temperature=0, max_tokens=4)),
        ("answer-n2", cell(n=2, temperature=0.8, seed=9, max_tokens=6)),
        ("follow-up-after-n2", _follow_up(MSGS, 18, 1, temperature=0, stream=True)),
    ]
    # P = SLOT_LEN - 3: a completion gets 3 tokens; the follow-up of a completion that filled its slot starts from 0, and its
    # prompt fills the whole slot, so it gets none
    long = _long_messages(tok_path, SLOT_LEN - 3)
    end = [
        ("end-n1-t0", dict(messages=long, temperature=0)),
        ("end-follow-up-after-n1", _follow_up(long, 0, 0, temperature=0)),
        ("end-n2-t0.8-seed-stream", dict(messages=long, n=2, temperature=0.8, seed=1, stream=True)),
        ("end-lp-k2-stream", dict(messages=long, logprobs=True, top_logprobs=2, stream=True)),
    ]
    return [("main", main), ("slot-end", end)]


def record(path=FIXTURE):
    sessions = []
    with tempfile.TemporaryDirectory() as d:
        stub = _build_stub(d)
        for name, cells in _matrix(stub[1]):
            responses, logs = _run_python(stub[1], [b for _, b in cells])
            done = [b(responses) if callable(b) else b for _, b in cells]   # the follow-ups as they were sent
            native, native_logs = _run_native(stub, done)
            out = []
            for (cname, _), body, r, log, nr, nlog in zip(cells, done, responses, logs, native, native_logs):
                c = {"name": cname, "request": body, "response": r, "log": log}
                if nr != r:
                    c["native_response"] = nr
                if nlog != log:
                    c["native_log"] = nlog
                out.append(c)
            sessions.append({"name": name, "cells": out})
    with open(path, "w", encoding="utf-8") as f:
        json.dump({"sessions": sessions}, f, indent=1)
        f.write("\n")


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    return _build_stub(str(tmp_path_factory.mktemp("api_parallel_paths")))


def _sessions():
    with open(FIXTURE, encoding="utf-8") as f:
        return json.load(f)["sessions"]


@pytest.mark.parametrize("server", ["python", "native"])
def test_servers_reproduce_the_recorded_parallel_completions(stub, server):
    for s in _sessions():
        bodies = [c["request"] for c in s["cells"]]
        if server == "python":
            got, logs = _run_python(stub[1], bodies)
            want, want_logs = [c["response"] for c in s["cells"]], [c["log"] for c in s["cells"]]
        else:
            got, logs = _run_native(stub, bodies)
            want = [c.get("native_response", c["response"]) for c in s["cells"]]
            want_logs = [c.get("native_log", c["log"]) for c in s["cells"]]
        for c, g, w, gl, wl in zip(s["cells"], got, want, logs, want_logs):
            assert g == w, (s["name"], c["name"])
            assert gl == wl, (s["name"], c["name"])


def test_slot_end_limits_of_the_fixture():
    """The recorded slot-end session gives every completion SLOT_LEN - P = 3 tokens, and the follow-up after the n = 1 answer,
    whose cache was cleared, prefills from 0 and gets none."""
    s = next(s for s in _sessions() if s["name"] == "slot-end")
    cells = {c["name"]: c for c in s["cells"]}
    assert cells["end-n1-t0"]["log"][0].split()[2:] == ["0", str(SLOT_LEN - 3)]
    assert json.loads(cells["end-n1-t0"]["response"])["usage"]["completion_tokens"] == 3
    follow = cells["end-follow-up-after-n1"]
    assert follow["log"][0].split()[2:] == ["0", str(SLOT_LEN)]
    assert json.loads(follow["response"])["usage"]["completion_tokens"] == 0


# ---- refusals ----------------------------------------------------------------------------------------------------------------

OK = dict(messages=MSGS, temperature=0, max_tokens=2)
# refused by both servers on both paths
BAD_BOTH = [dict(messages=MSGS, temperature=-0.5), [OK]]
# wrong field shapes: refused by the Python server (the native server reads a non-numeric number as absent)
BAD_SHAPES = [dict(messages=MSGS, temperature=None), dict(messages=MSGS, max_tokens=None), dict(messages=MSGS, top_p=None),
              dict(messages=MSGS, temperature="0.5"), dict(messages=MSGS, max_tokens="3"), dict(messages=MSGS, seed=None),
              dict(messages=MSGS, seed="3"), dict(messages="hello"), dict(messages=["hello"]), dict(messages=[{"role": "user"}]),
              dict(messages=[{"role": "user", "content": None}]), dict(messages={"role": "user", "content": "hi"}), [1], "hello", 3]


def _refusals(post_all, bad):
    bodies = [x for b in bad for x in (b, OK)]
    out = post_all(bodies)
    for i in range(0, len(bodies), 2):
        assert out[i] == "", bodies[i]                                          # closed without a response
        assert json.loads(out[i + 1])["usage"]["completion_tokens"] == 2, bodies[i]


@pytest.mark.parametrize("parallel", [1, PARALLEL])
def test_python_server_refuses_malformed_bodies_and_keeps_serving(stub, parallel):
    def post_all(bodies):
        port, _, join = _python_server(stub[1], len(bodies), parallel, seq_len=4096)
        out = [tsc._post(port, b) for b in bodies]
        join()
        return out
    _refusals(post_all, BAD_BOTH + BAD_SHAPES)


@pytest.mark.parametrize("parallel", [1, PARALLEL])
def test_native_server_refuses_malformed_bodies_and_keeps_serving(stub, tmp_path, parallel):
    if parallel == 1:   # the single-sequence path over the stub of tests/test_api_completion_paths.py
        from test_api_completion_paths import _build_stub as build_single
        exe, tok = build_single(str(tmp_path))
        server, args = (exe, tok), ["12", "4096"]
    else:
        server, args = stub, [str(PARALLEL), "10", "0"]

    def post_all(bodies):
        port, log = _native_server(server, len(bodies), args)
        try:
            return [tsc._post(port, b) for b in bodies]
        finally:
            log()
    _refusals(post_all, BAD_BOTH)


if __name__ == "__main__":
    record()
