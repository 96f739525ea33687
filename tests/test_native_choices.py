"""`n` completions in both API servers on CPU: the native server (csrc/app/api_server.cpp, over tests/native/api_choices_stub_main.cpp)
and the Python one (apps/api_server.py, over the same stub model in Python) must return identical JSON and streamed text."""
import http.client
import json
import os
import re
import socket
import subprocess
import threading
import time
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    d = tmp_path_factory.mktemp("api_stub_choices")
    exe = str(d / "api_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_choices_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = str(d / "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


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


def _post(port, body):
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=20)
    try:
        c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
        r = c.getresponse()
        return r.read()
    except (http.client.RemoteDisconnected, ConnectionError):
        return None
    finally:
        c.close()


def _norm(raw: bytes):
    """JSON without the timestamp, or the list of streamed events without timestamps."""
    text = raw.decode("utf-8")
    if text.lstrip().startswith("{"):
        j = json.loads(text)
        j.pop("created")
        return j
    events = [e for e in text.split("\r\n\r\n") if e.startswith("data: ")]
    out = []
    for e in events:
        if e == "data: [DONE]":
            out.append(e)
        else:
            j = json.loads(e[6:])
            j.pop("created")
            out.append(j)
    return out


MSGS = [{"role": "system", "content": "be brief"}, {"role": "user", "content": "héllo ✓"}]


def test_python_and_native_servers_agree_on_choices(stub):
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args

    exe, tok_path = stub
    H = host()
    tok = H.Tokenizer(tok_path)
    regular, eos = tok.regular_vocab_size, list(tok.eos_ids)[0]
    py_log = []

    class FakeInference:
        """tests/native/api_choices_stub_main.cpp in Python (the greedy branch emits EOS after 12 tokens)."""
        comm = None

        def __init__(self):
            self.produced = 0

        def prefill(self, tokens, pos):
            py_log.append((pos, len(tokens)))
            self.produced = 0
            self.end = pos + len(tokens)

        def next_token(self, token, pos, sampler):
            if sampler.temperature > 0:
                if pos + 1 - self.end > 12:
                    return eos
                return (token * 7 + pos * 13 + 5 + (sampler.seed % 997) * 31) % regular
            self.produced += 1
            return eos if self.produced > 12 else (token * 7 + pos * 13 + 5) % regular

        next_token_at = next_token

        def forget_device_seed(self):
            pass

        def save_sampler(self):
            return None

        def restore_sampler(self, saved):
            pass

        def batched_choices(self, n):
            return False

    n_req = 8   # readiness probe + 7 requests
    port_py = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port_py), "--temperature", "0"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=FakeInference(), tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                          header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, n_req), daemon=True)
    th.start()
    _wait(port_py)
    port_nat = _free_port()
    proc = subprocess.Popen([exe, tok_path, str(port_nat), str(n_req)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    _wait(port_nat)
    results = {}
    try:
        base = {"messages": MSGS, "temperature": 0.8, "max_tokens": 9, "seed": 42}
        for name, body in (("json", dict(base, n=3)), ("stream", dict(base, n=3, stream=True))):
            results[name] = [_post(port_py, body), _post(port_nat, body)]
        answer = json.loads(results["json"][0])["choices"][1]["message"]["content"]
        follow = MSGS + [{"role": "assistant", "content": answer}, {"role": "user", "content": "more"}]
        results["follow"] = [_post(port_py, {"messages": follow, "temperature": 0, "max_tokens": 4}),
                             _post(port_nat, {"messages": follow, "temperature": 0, "max_tokens": 4})]
        for bad in (0, 9, "x"):
            assert _post(port_py, dict(base, n=bad)) in (None, b"") and _post(port_nat, dict(base, n=bad)) in (None, b"")
        results["plain"] = [_post(port_py, {"messages": [{"role": "user", "content": "fresh"}], "temperature": 0, "max_tokens": 64}),
                            _post(port_nat, {"messages": [{"role": "user", "content": "fresh"}], "temperature": 0, "max_tokens": 64})]
    finally:
        try:
            out, _ = proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            out, _ = proc.communicate()
        th.join(timeout=20)
    for name, (a, b) in results.items():
        assert _norm(a) == _norm(b), name
    j = _norm(results["json"][0])
    assert [c["index"] for c in j["choices"]] == [0, 1, 2] and len({c["message"]["content"] for c in j["choices"]}) == 3
    assert j["usage"]["completion_tokens"] == 27 and j["usage"]["total_tokens"] == j["usage"]["prompt_tokens"] + 27
    ev = _norm(results["stream"][0])
    assert ev[-1] == "data: [DONE]" and ev.count("data: [DONE]") == 1
    assert [e["choices"][0]["index"] for e in ev[:-1] if e["choices"][0]["finish_reason"] == "stop"] == [0, 1, 2]
    streamed = ["".join(e["choices"][0]["delta"]["content"] for e in ev[:-1] if "delta" in e["choices"][0] and e["choices"][0]["index"] == i)
                for i in range(3)]
    assert streamed == [c["message"]["content"] for c in j["choices"]]
    plain = _norm(results["plain"][0])
    assert len(plain["choices"]) == 1 and plain["usage"]["completion_tokens"] == 13
    # the follow-up quoting choice 1 prefills from the prompt end of the first request (the stub logs "POS start n")
    nat = [(int(a), int(b)) for a, b in re.findall(r"POS (\d+) (\d+)", out)]
    assert py_log == nat
    first_end = nat[0][0] + nat[0][1]
    assert nat[2][0] == first_end and nat[2][0] > 0
    assert "🐤 Found naive cache for 2 messages" in out
