"""Both API servers answer every chat completion, with or without `n`, through one path. A fixed request matrix over the
deterministic stub model (tests/native/api_choices_stub_main.cpp, and StubModel below, its twin in Python) was recorded from the
Python server before the n = 1 and n >= 2 paths were merged; both servers must still reproduce every response byte for byte,
apart from `created`, and make the same prefills ("POS <start> <n>").

Re-record with `python tests/test_api_completion_paths.py`: it runs the matrix against the Python server in this tree and against
the native stub, and keeps the native answer of any cell where the two servers disagree under "native_response"."""
import http.client
import json
import os
import re
import socket
import subprocess
import sys
import tempfile
import threading
import time
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "api_completions.json")
MSGS = [{"role": "system", "content": "be brief"}, {"role": "user", "content": "héllo ✓"}]


class StubModel:
    """tests/native/api_choices_stub_main.cpp in Python."""
    comm = None

    def __init__(self, regular: int, eos: int, eos_after: int = 12):
        self.regular, self.eos, self.eos_after = regular, eos, eos_after
        self.produced = self.end = 0
        self.log = []

    def prefill(self, tokens, pos):
        self.log.append([pos, len(tokens)])
        self.produced = 0
        self.end = pos + len(tokens)

    def next_token(self, token, pos, sampler):
        if sampler.temperature > 0:
            if pos + 1 - self.end > self.eos_after:
                return self.eos
            return (token * 7 + pos * 13 + 5 + (sampler.seed % 997) * 31) % self.regular
        self.produced += 1
        return self.eos if self.produced > self.eos_after else (token * 7 + pos * 13 + 5) % self.regular

    def forget_device_seed(self):
        pass

    def save_sampler(self):
        return None

    def restore_sampler(self, saved):
        pass

    def batched_choices(self, n):
        return False


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _wait(port):
    for _ in range(200):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            return
        except OSError:
            time.sleep(0.05)


def _post(port, body) -> str:
    """The response body (chunked framing undone) without its `created` stamps."""
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=20)
    try:
        c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
        raw = c.getresponse().read()
    finally:
        c.close()
    return re.sub(r'"created": \d+, ', "", raw.decode("utf-8", errors="surrogateescape"))   # the native server sends bytes as decoded


def _build_stub(d):
    exe = os.path.join(d, "api_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_choices_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


def _run_python(tok_path, seq_len, bodies):
    """Serves `bodies` one after another on the Python server over StubModel: (responses, prefills)."""
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args

    H = host()
    tok = H.Tokenizer(tok_path)
    model = StubModel(tok.regular_vocab_size, list(tok.eos_ids)[0])
    port = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                          header=SimpleNamespace(seq_len=seq_len, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, len(bodies) + 1), daemon=True)   # + the readiness probe
    th.start()
    _wait(port)
    out = []
    for b in bodies:
        out.append(_post(port, b(out) if callable(b) else b))
    th.join(timeout=20)
    return out, model.log


def _run_native(stub, seq_len, bodies):
    exe, tok_path = stub
    port = _free_port()
    proc = subprocess.Popen([exe, tok_path, str(port), str(len(bodies) + 1), "12", str(seq_len)], stdout=subprocess.PIPE,
                            stderr=subprocess.STDOUT, text=True)
    try:
        _wait(port)
        out = [_post(port, b) for b in bodies]
    finally:
        try:
            log, _ = proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            log, _ = proc.communicate()
    return out, [[int(a), int(b)] for a, b in re.findall(r"POS (\d+) (\d+)", log)]


def _follow_up(answer: int, choice: int, **extra):
    """A history that quotes choice `choice` of response `answer` of the same session."""
    def body(prev):
        j = json.loads(prev[answer])
        msgs = MSGS + [{"role": "assistant", "content": j["choices"][choice]["message"]["content"]}, {"role": "user", "content": "more"}]
        return dict(extra, messages=msgs)
    return body


def _matrix():
    """(session name, cells): each cell is (name, body or body-builder over the earlier responses by index)."""
    def cell(**kw):
        return dict(kw, messages=MSGS)
    main = [
        ("n-absent-t0", cell(temperature=0)),
        ("n-absent-t0-stream-max4", cell(temperature=0, stream=True, max_tokens=4)),
        ("n-absent-t0.8-noseed-max4", cell(temperature=0.8, max_tokens=4)),
        ("n1-t0.8-seed-max4", cell(n=1, temperature=0.8, seed=42, max_tokens=4)),
        ("n1-t0.8-noseed-stream", cell(n=1, temperature=0.8, stream=True)),
        ("n1-t0-max4", cell(n=1, temperature=0, max_tokens=4)),
        ("n2-t0.8-seed", cell(n=2, temperature=0.8, seed=7)),
        ("n2-t0-stream-max4", cell(n=2, temperature=0, stream=True, max_tokens=4)),
        ("n3-t0.8-noseed-max4", cell(n=3, temperature=0.8, max_tokens=4)),
        ("n3-t0.8-seed-stream", cell(n=3, temperature=0.8, seed=42, stream=True)),
        ("n3-t0", cell(n=3, temperature=0)),
        ("n8-t0.8-seed-max4", cell(n=8, temperature=0.8, seed=5, max_tokens=4)),
        ("n8-t0.8-noseed-stream-max4", cell(n=8, temperature=0.8, stream=True, max_tokens=4)),
        ("n8-t0", cell(n=8, temperature=0)),
        ("n-absent-t0.8-seed-answer", cell(temperature=0.8, seed=3, max_tokens=6)),
        ("follow-up-after-n1", _follow_up(14, 0, temperature=0, max_tokens=4)),
        ("n3-t0.8-seed-answer", cell(n=3, temperature=0.8, seed=9, max_tokens=6)),
        ("follow-up-after-n3", _follow_up(16, 2, temperature=0, stream=True)),
    ]
    # seq_len = P + 5 (P: the prompt's last position): n = 1 gets 5 tokens, n = 2 gets 2 per choice, n = 3 gets 1
    end = [
        ("end-n1", cell(temperature=0)),
        ("end-follow-up-after-n1", _follow_up(0, 0, temperature=0)),
        ("end-n2-t0.8-seed", cell(n=2, temperature=0.8, seed=1)),
        ("end-n3-t0.8-seed-stream", cell(n=3, temperature=0.8, seed=1, stream=True)),
        ("end-n1-t0.8-seed-stream", cell(temperature=0.8, seed=1, stream=True)),
    ]
    return [("main", main), ("context-end", end)]


def record(path=FIXTURE):
    sessions = []
    with tempfile.TemporaryDirectory() as d:
        stub = _build_stub(d)
        seq_len = 4096
        for name, cells in _matrix():
            if name == "context-end":
                seq_len = sessions[0]["prefills"][0][1] + 5
            responses, prefills = _run_python(stub[1], seq_len, [b for _, b in cells])
            done = [b(responses) if callable(b) else b for _, b in cells]   # the follow-ups as they were sent
            native, native_prefills = _run_native(stub, seq_len, done)
            out = []
            for (cname, _), body, r, nr in zip(cells, done, responses, native):
                c = {"name": cname, "request": body, "response": r}
                if nr != r:
                    c["native_response"] = nr
                out.append(c)
            s = {"name": name, "seq_len": seq_len, "cells": out, "prefills": prefills}
            if native_prefills != prefills:
                s["native_prefills"] = native_prefills
            sessions.append(s)
    with open(path, "w", encoding="utf-8") as f:
        json.dump({"sessions": sessions}, f, indent=1)
        f.write("\n")


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    return _build_stub(str(tmp_path_factory.mktemp("api_paths")))


def _sessions():
    with open(FIXTURE, encoding="utf-8") as f:
        return json.load(f)["sessions"]


@pytest.mark.parametrize("server", ["python", "native"])
def test_servers_reproduce_the_recorded_completions(stub, server):
    for s in _sessions():
        bodies = [c["request"] for c in s["cells"]]
        if server == "python":
            got, prefills = _run_python(stub[1], s["seq_len"], bodies)
            want, want_prefills = [c["response"] for c in s["cells"]], s["prefills"]
        else:
            got, prefills = _run_native(stub, s["seq_len"], bodies)
            want = [c.get("native_response", c["response"]) for c in s["cells"]]
            want_prefills = s.get("native_prefills", s["prefills"])
        for c, g, w in zip(s["cells"], got, want):
            assert g == w, (s["name"], c["name"])
        assert prefills == want_prefills, s["name"]


def test_context_end_limits_of_the_fixture():
    """The recorded context-end session gives n = 1 seq_len - P tokens and n >= 2 floor((seq_len - 1 - P) / n) per choice, and
    the follow-up after the n = 1 answer prefills from 0 because that answer filled the context."""
    s = next(s for s in _sessions() if s["name"] == "context-end")
    cells = {c["name"]: c for c in s["cells"]}
    P = s["prefills"][0][1]
    assert s["seq_len"] == P + 5
    assert json.loads(cells["end-n1"]["response"])["usage"]["completion_tokens"] == 5
    assert json.loads(cells["end-n2-t0.8-seed"]["response"])["usage"]["completion_tokens"] == 2 * 2
    assert s["prefills"][1][0] == 0


def test_run_choices_single_sequence_limit():
    """run_choices(n=1) stops at the end of the context like the single-sequence loops: seq_len - P tokens."""
    from distributed_llama_b200 import host
    from distributed_llama_b200.api import run_choices

    H = host()

    class Backend:
        def next_token(self, token, pos, sampler):
            return 7

    for seq_len, P, max_tokens, want in ((18, 13, -1, 5), (18, 13, 3, 3), (18, 13, 9, 5), (18, 17, -1, 1), (18, 18, -1, 0), (18, 13, 0, 5)):
        out = run_choices(Backend(), 1, P, 1, max_tokens, seq_len, H.Sampler(512, 0.0, 0.9, 1), 0, lambda i, t: False)
        assert [len(o) for o in out] == [want], (seq_len, P, max_tokens)
    # n >= 2 keeps its share of the rows after P: floor((seq_len - 1 - P) / n)
    out = run_choices(Backend(), 1, 13, 2, -1, 18, H.Sampler(512, 0.0, 0.9, 1), 0, lambda i, t: False)
    assert [len(o) for o in out] == [2, 2]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    record()
