"""`--parallel N` in the native API server on the CPU (tests/native/api_parallel_stub_main.cpp over the real csrc/app/api_server.cpp),
and the same completions from the Python server (tests/test_api_parallel.py's SlotStub is the stub's twin)."""
import http.client
import json
import os
import re
import socket
import subprocess
import threading

import pytest

from test_api_parallel import BODIES, SlotStub, _concurrent, _free_port, _msgs, _post

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("api_parallel"))
    exe = os.path.join(d, "api_parallel_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_parallel_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe, "-lpthread"], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


class Native:
    def __init__(self, stub, max_requests, parallel=4, eos_after=10, delay_ms=20):
        exe, tok = stub
        self.port = _free_port()
        self.proc = subprocess.Popen([exe, tok, str(self.port), str(max_requests + 1), str(parallel), str(eos_after), str(delay_ms)],
                                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        for _ in range(200):
            try:
                socket.create_connection(("127.0.0.1", self.port), timeout=0.2).close()   # the readiness probe
                break
            except OSError:
                import time
                time.sleep(0.02)

    def log(self):
        try:
            out, _ = self.proc.communicate(timeout=30)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            out, _ = self.proc.communicate()
        return out


def test_native_concurrent_requests_match_alone(stub):
    srv = Native(stub, 2 * len(BODIES))
    alone = [_post(srv.port, b) for b in BODIES]
    together, stamps = _concurrent(srv.port, BODIES, stagger=0.005)
    srv.log()
    assert together == alone                                 # the fifth request queued and completed
    assert stamps[1][0] < stamps[0][-1]                      # B's first chunk arrived before A's last


def test_native_disconnect_malformed_and_too_many_choices(stub):
    srv = Native(stub, 3 + 3 + 3, eos_after=30, delay_ms=30)
    bodies = BODIES[:3]
    alone = [_post(srv.port, b) for b in bodies]

    def quitter():
        s = socket.create_connection(("127.0.0.1", srv.port))
        body = json.dumps(dict(messages=_msgs(9), stream=True)).encode()
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nContent-Length: " + str(len(body)).encode() + b"\r\n\r\n" + body)
        s.recv(64)
        s.close()

    def refused(payload):
        s = socket.create_connection(("127.0.0.1", srv.port))
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nContent-Length: " + str(len(payload)).encode() + b"\r\n\r\n" + payload)
        assert s.recv(64) == b""                             # closed without a response
        s.close()
    side = [threading.Thread(target=quitter), threading.Thread(target=refused, args=(b"{not json",)),
            threading.Thread(target=refused, args=(json.dumps(dict(messages=_msgs(1), n=5, temperature=0.8)).encode(),))]
    for t in side:
        t.start()
    together, _ = _concurrent(srv.port, bodies)
    for t in side:
        t.join(timeout=30)
    srv.log()
    assert together == alone


def _sequence():
    """Requests sent one after another: plain, streamed, seeded, n = 2 sampled, n = 3 greedy, and follow-ups."""
    return [dict(messages=_msgs(0)), dict(messages=_msgs(1), stream=True, max_tokens=4), dict(messages=_msgs(2), temperature=0.8, seed=42),
            dict(messages=_msgs(3), n=2, temperature=0.8, seed=7), dict(messages=_msgs(3), n=3, temperature=0),
            dict(messages=_msgs(4), temperature=0.8), "follow-up"]


def _run(port, bodies):
    out = []
    for b in bodies:
        if b == "follow-up":
            b = dict(messages=_msgs(4) + [{"role": "assistant", "content": out[-1][0]}, {"role": "user", "content": "more"}])
        out.append(_post(port, b))
    return out


def test_python_and_native_servers_agree(stub, tmp_path):
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    from types import SimpleNamespace
    bodies = _sequence()
    srv = Native(stub, len(bodies))
    native = _run(srv.port, bodies)
    native_pos = [tuple(int(x) for x in m) for m in re.findall(r"POS (\d+) (\d+) (\d+)", srv.log())]

    H = host()
    tok = H.Tokenizer(stub[1])
    model = SlotStub(4, 256, tok.regular_vocab_size, list(tok.eos_ids)[0], 10, 0.02)
    port = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", stub[1], "--host", "127.0.0.1", "--port", str(port), "--temperature", "0",
                       "--parallel", "4"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 77),
                          header=SimpleNamespace(seq_len=1024, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, len(bodies) + 1), daemon=True)
    th.start()
    for _ in range(200):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            break
        except OSError:
            import time
            time.sleep(0.02)
    python = _run(port, bodies)
    th.join(timeout=30)
    assert python == native
    assert [p for p in model.prefills] == native_pos
    assert native_pos[-1][1] > 0                             # the follow-up re-used its slot's prompt cache


@pytest.mark.parametrize("argv,env", [(["--parallel", "0"], {}), (["--parallel", "9"], {}), (["--parallel", "2", "--gpus", "2"], {}),
                                      (["--parallel", "2", "--workers", "10.0.0.2:9999"], {}),
                                      (["--parallel", "2"], {"DL_COLLECTIVES": "nccl"}), (["--parallel", "2"], {"DL_HOST_SAMPLER": "1"})])
def test_native_startup_refusals(argv, env):
    exe = os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")
    if not os.path.exists(exe):
        from distributed_llama_b200 import _build
        _build.build_all(verbose=False)
    env = {k: v for k, v in os.environ.items() if k not in ("DL_COLLECTIVES", "DL_HOST_SAMPLER")} | env
    r = subprocess.run([exe, "--model", "m.m", "--tokenizer", "t.t"] + argv, capture_output=True, text=True, env=env, timeout=30)
    assert r.returncode == 1
    assert "--parallel" in r.stderr and len(r.stderr.strip().splitlines()) == 1
