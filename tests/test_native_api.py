"""Native API server (csrc/app/api_server.cpp) end to end on CPU: real sockets, HTTP parsing, JSON in/out, chat template, stop
detection, SSE streaming and NaiveCache prefix re-use over a deterministic stub model (tests/native/api_choices_stub_main.cpp)."""
import http.client
import json
import os
import socket
import subprocess
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    d = tmp_path_factory.mktemp("api_stub")
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


def _start(stub, n_requests, eos_after=12):
    exe, tok = stub
    port = _free_port()
    proc = subprocess.Popen([exe, tok, str(port), str(n_requests), str(eos_after)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    for _ in range(100):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            break
        except OSError:
            time.sleep(0.05)
    return proc, port


def _req(port, method, path, body=None):
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=20)
    c.request(method, path, body=json.dumps(body) if body is not None else None,
              headers={"Content-Type": "application/json"} if body is not None else {})
    r = c.getresponse()
    data = r.read()
    c.close()
    return r.status, dict(r.getheaders()), data


def test_routes_json_stream_and_cache(stub):
    # the readiness probe in _start consumes one request slot (an empty connection is logged as a socket error)
    proc, port = _start(stub, 7)
    try:
        st, hdr, _ = _req(port, "OPTIONS", "/v1/chat/completions")
        assert st == 204 and hdr["Access-Control-Allow-Origin"] == "*"
        st, _, data = _req(port, "GET", "/v1/models")
        assert st == 200 and json.loads(data)["data"][0]["id"] == "stub.m"
        st, _, data = _req(port, "GET", "/nope")
        assert st == 404 and data == b"Not Found"
        msgs = [{"role": "system", "content": "You are \"terse\".\n"}, {"role": "user", "content": "héllo wörld ✓"}]
        st, hdr, data = _req(port, "POST", "/v1/chat/completions", {"messages": msgs, "temperature": 0, "max_tokens": 64})
        assert st == 200 and hdr["Content-Type"].startswith("application/json")
        j = json.loads(data)
        assert j["object"] == "chat.completion" and j["choices"][0]["finish_reason"] == "stop"
        answer = j["choices"][0]["message"]["content"]
        u = j["usage"]
        assert u["completion_tokens"] == 13 and u["total_tokens"] == u["prompt_tokens"] + 13     # 12 tokens + the EOS step
        # streamed follow-up that extends the history -> NaiveCache restarts after the cached turns
        msgs2 = msgs + [{"role": "assistant", "content": answer}, {"role": "user", "content": "again"}]
        st, hdr, data = _req(port, "POST", "/v1/chat/completions", {"messages": msgs2, "stream": True, "temperature": 0})
        assert st == 200 and hdr["Content-Type"].startswith("text/event-stream")      # http.client already undid the chunked framing
        events = [e for e in data.decode("utf-8").split("\r\n\r\n") if e.startswith("data: ")]
        assert events[-1] == "data: [DONE]"
        chunks = [json.loads(e[6:]) for e in events[:-1]]
        assert chunks[-1]["choices"][0]["finish_reason"] == "stop" and "delta" not in chunks[-1]["choices"][0]
        text = "".join(c["choices"][0]["delta"]["content"] for c in chunks[:-1])
        assert all(c["choices"][0]["delta"]["role"] == "assistant" for c in chunks[:-1]) and isinstance(text, str)
        # a history that does not extend the cache clears it
        st, _, data = _req(port, "POST", "/v1/chat/completions", {"messages": [{"role": "user", "content": "fresh"}], "temperature": 0})
        assert st == 200
    finally:
        try:
            out, _ = proc.communicate(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
            out, _ = proc.communicate()
    import re
    starts = [int(m.group(1)) for m in re.finditer(r"POS (\d+) (\d+)", out)]
    assert len(starts) == 3 and starts[0] == 0 and starts[1] > 0 and starts[2] == 0, out[-1500:]
    assert "🐤 Found naive cache for 3 messages" in out
    assert "⭐ Chat template: llama3" in out


def test_bad_requests_do_not_kill_the_server(stub):
    proc, port = _start(stub, 4)
    try:
        s = socket.create_connection(("127.0.0.1", port))
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nContent-Length: 9\r\n\r\n{not json")
        s.settimeout(5)
        assert s.recv(100) == b""            # connection closed without a response, server logs the error
        s.close()
        st, _, _ = _req(port, "POST", "/v1/chat/completions", {"nomessages": 1})
        assert st is not None
    except (http.client.RemoteDisconnected, ConnectionError):
        pass
    st, _, data = _req(port, "GET", "/v1/models")
    assert st == 200
    out, _ = proc.communicate(timeout=10)
    assert "JSON parse error" in out and "missing key" in out


def test_json_reader_writer(tmp_path):
    exe = str(tmp_path / "json_test")
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", os.path.join(ROOT, "tests", "native", "json_test.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "JSON_TEST_OK" in r.stdout, r.stdout


def test_python_and_native_servers_agree(stub):
    """The Python server (apps/api_server.py, used for multi-GPU serving) and the native one run the same deterministic stub
    model: their non-stream JSON and their streamed text must be identical for the same requests."""
    import threading
    from types import SimpleNamespace

    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args

    exe, tok_path = stub
    H = host()
    tok = H.Tokenizer(tok_path)
    regular, eos = tok.regular_vocab_size, list(tok.eos_ids)[0]

    class FakeInference:
        comm = None

        def __init__(self):
            self.produced = 0

        def prefill(self, tokens, pos):
            self.produced = 0

        def forward_greedy(self, token, pos):
            self.produced += 1
            return eos if self.produced > 12 else (token * 7 + pos * 13 + 5) % regular

        def next_token(self, token, pos, sampler):
            return self.forward_greedy(token, pos)

    port_py = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port_py), "--temperature", "0"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=FakeInference(), tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 1),
                          header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, 2), daemon=True)
    th.start()
    for _ in range(100):
        try:
            socket.create_connection(("127.0.0.1", port_py), timeout=0.2).close()
            break
        except OSError:
            time.sleep(0.05)
    # the probe above consumed one of the two request slots of the Python server; the native stub gets 1 probe + 1 request
    proc, port_nat = _start(stub, 2)
    msgs = [{"role": "system", "content": "be brief"}, {"role": "user", "content": "héllo ✓ \"quoted\""}]
    body = {"messages": msgs, "temperature": 0, "max_tokens": 64}
    try:
        _, _, a = _req(port_py, "POST", "/v1/chat/completions", body)
        _, _, b = _req(port_nat, "POST", "/v1/chat/completions", body)
    finally:
        try:
            proc.communicate(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
        th.join(timeout=10)
    ja, jb = json.loads(a), json.loads(b)
    for j in (ja, jb):
        j.pop("created")
    assert ja == jb and ja["usage"]["completion_tokens"] == 13


def test_example_client_against_native_server(stub, capsys):
    """examples/chat_api_client.py (non-stream + stream helpers) talks to the native server."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("chat_api_client", os.path.join(ROOT, "examples", "chat_api_client.py"))
    client = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(client)
    proc, port = _start(stub, 3)
    client.HOST = f"http://127.0.0.1:{port}"
    try:
        out = client.chat([{"role": "user", "content": "2+2?"}], max_tokens=32)
        assert out["choices"][0]["message"]["role"] == "assistant" and out["usage"]["completion_tokens"] == 13
        client.chat([{"role": "user", "content": "and 3+3?"}], max_tokens=32, stream=True)
        streamed = capsys.readouterr().out
        assert len(streamed.strip()) > 0
    finally:
        try:
            proc.communicate(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
