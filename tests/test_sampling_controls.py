"""Sampling controls: presence / frequency penalties and logit bias (host Sampler, both API servers).

* The host Sampler's transform against a numpy float32 reference of the formula, bit for bit, and its draws: a +100 bias always
  wins greedy decoding, -100 never does, a large frequency penalty moves greedy decoding off a token once it has been drawn, and
  the counts start from zero for every completion.
* Both servers over stub models that draw with the sampler they are handed (tests/native/api_controls_stub_main.cpp and
  ControlsStub below, its Python twin) and log the controls each completion starts with: identical responses and logs for a
  matrix of valid requests; every malformed value is refused with the server still answering; zero penalties and an empty
  logit_bias answer exactly as a request without them.
"""
import json
import os
import re
import socket
import subprocess
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MSGS = [{"role": "system", "content": "be brief"}, {"role": "user", "content": "hello"}]


def _H():
    from distributed_llama_b200 import host
    return host()


def reference_transform(logits, counts, bias, presence, frequency):
    """The controls' formula in numpy float32: x = l + bias (if any); where c > 0: x = x - c * frequency, then x = x - presence."""
    x = np.asarray(logits, dtype=np.float32).copy()
    if bias:
        b = np.zeros_like(x)
        for t, v in bias:
            b[t] = np.float32(v)
        x = x + b
    hit = counts > 0
    pen = counts[hit].astype(np.float32) * np.float32(frequency)
    x[hit] = (x[hit] - pen) - np.float32(presence)
    return x


def _draw_counts(smp, V, tokens):
    """Makes `smp` draw `tokens` (greedy over one-hot logits that dominate any control) so that its counts become known."""
    for t in tokens:
        lg = np.zeros(V, dtype=np.float32)
        lg[t] = 1e6
        assert smp.sample(lg) == t


@pytest.mark.parametrize("V", [1000, 32003])
def test_transform_matches_reference_bit_for_bit(V):
    H = _H()
    rs = np.random.RandomState(V)
    for presence, frequency, nb in ((0.5, 1.25, 30), (-2.0, 2.0, 100), (1.7, -0.3, 0), (0.0, 0.0, 7), (0.1, 0.0, 0)):
        bias = sorted({int(t): float(np.float32(v)) for t, v in zip(rs.randint(0, V, nb), rs.uniform(-100, 100, nb))}.items())
        smp = H.Sampler(V, 0.0, 0.9, 1)
        smp.set_controls(presence, frequency, bias)
        assert smp.controls_active
        drawn = [int(t) for t in rs.randint(0, V, 200)]
        _draw_counts(smp, V, drawn)
        counts = np.bincount(drawn, minlength=V).astype(np.uint32)
        assert np.array_equal(np.asarray(smp.counts), counts)
        lg = (rs.randn(V) * 4).astype(np.float32)
        got = np.asarray(smp.apply_controls(lg))
        want = reference_transform(lg, counts, bias, presence, frequency)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_bias_and_penalties_steer_greedy_decoding():
    H = _H()
    V = 512
    rs = np.random.RandomState(3)
    up = H.Sampler(V, 0.0, 0.9, 1)
    up.set_controls(0.0, 0.0, [(77, 100.0)])
    down = H.Sampler(V, 0.0, 0.9, 1)
    down.set_controls(0.0, 0.0, [(5, -100.0)])
    for _ in range(200):
        lg = (rs.randn(V) * 10).astype(np.float32)
        assert up.sample(lg) == 77
        lg[5] = lg.max() + 50.0            # the unbiased arg-max, by a margin below 100
        assert down.sample(lg) != 5
    # a frequency penalty moves greedy decoding off a token once it has been drawn
    fp = H.Sampler(V, 0.0, 0.9, 1)
    fp.set_controls(0.0, 2.0, [])
    lg = np.zeros(V, dtype=np.float32)
    lg[9], lg[4] = 3.0, 2.0
    assert [fp.sample(lg) for _ in range(3)] == [9, 4, 9]   # 3 - 2 = 1 < 2; then 2 - 2 = 0 < 1; then 9 again (3 - 2 = 1 > 0)
    # sampled draws (temperature > 0) count as well, and counts restart at zero for every completion
    s = H.Sampler(V, 0.8, 0.9, 5)
    s.set_controls(0.5, 0.0, [])
    gen = s.completion_generation
    for _ in range(10):
        s.sample((rs.randn(V)).astype(np.float32))
    assert int(np.asarray(s.counts).sum()) == 10
    s.begin_completion()
    assert int(np.asarray(s.counts).sum()) == 0 and s.completion_generation != gen
    # a fresh sampler never shares a completion generation with another one
    assert len({H.Sampler(V, 0.8, 0.9, 5).completion_generation for _ in range(5)}) == 5


def test_controls_off_draw_exactly_as_before():
    H = _H()
    V = 4096
    rs = np.random.RandomState(8)
    for T, topp in ((0.0, 0.9), (0.8, 0.9), (1.3, 0.0)):
        a, b = H.Sampler(V, T, topp, 99), H.Sampler(V, T, topp, 99)
        b.set_controls(0.0, 0.0, [])
        assert not b.controls_active
        for _ in range(50):
            lg = (rs.randn(V) * 3).astype(np.float32)
            assert a.sample(lg) == b.sample(lg)
        assert len(b.counts) == 0


def test_sampler_refuses_ids_outside_the_vocabulary():
    H = _H()
    s = H.Sampler(100, 0.0, 0.9, 1)
    for bad in ([(100, 1.0)], [(-1, 1.0)]):
        with pytest.raises(ValueError):
            s.set_controls(0.0, 0.0, bad)


# ---- both servers --------------------------------------------------------------------------------------------------------------


class ControlsStub:
    """tests/native/api_controls_stub_main.cpp in Python."""
    comm = None

    def __init__(self, V: int, eos: int, eos_after: int = 12):
        self.V, self.eos, self.eos_after = V, eos, eos_after
        self.end = 0
        self.last = None
        self.log = []
        self.t_hash = (np.arange(V, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)

    def prefill(self, tokens, pos):
        self.log.append(f"POS {pos} {len(tokens)}")
        self.end = pos + len(tokens)

    def next_token(self, token, pos, sampler):
        if sampler.completion_generation != self.last:
            self.last = sampler.completion_generation
            self.log.append(" ".join([f"CTL {sampler.presence_penalty:.9g} {sampler.frequency_penalty:.9g}"] +
                                     [f"{t}:{v:.9g}" for t, v in sampler.logit_bias]))
        if pos + 1 - self.end > self.eos_after:
            return self.eos
        k = ((self.t_hash[:sampler.vocab_size] + np.uint64(token * 97 + pos * 13)) & np.uint64(0xFFFFFFFF)) % np.uint64(1000)
        lg = k.astype(np.float32) / np.float32(100.0)
        return int(sampler.sample(lg))

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
    """The response body without its `created` stamps; "" when the server closed the connection without answering."""
    data = json.dumps(body).encode() if not isinstance(body, bytes) else body
    req = (b"POST /v1/chat/completions HTTP/1.1\r\nHost: x\r\nContent-Type: application/json\r\nContent-Length: " +
           str(len(data)).encode() + b"\r\n\r\n" + data)
    with socket.create_connection(("127.0.0.1", port), timeout=20) as c:
        c.sendall(req)
        raw = b""
        while True:
            chunk = c.recv(65536)
            if not chunk:
                break
            raw += chunk
    if not raw:
        return ""
    head, _, rest = raw.partition(b"\r\n\r\n")
    if b"chunked" in head:
        out, r = b"", rest
        while r:
            size, _, r = r.partition(b"\r\n")
            n = int(size, 16)
            if n == 0:
                break
            out += r[:n]
            r = r[n + 2:]
        rest = out
    return re.sub(r'"created": \d+, ', "", rest.decode("utf-8", errors="surrogateescape"))


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("api_controls"))
    exe = os.path.join(d, "api_controls_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_controls_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


def _run_python(tok_path, bodies):
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    H = _H()
    tok = H.Tokenizer(tok_path)
    model = ControlsStub(tok.vocab_size, list(tok.eos_ids)[0])
    port = _free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                          header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, len(bodies) + 1), daemon=True)   # + the readiness probe
    th.start()
    _wait(port)
    out = [_post(port, b) for b in bodies]
    th.join(timeout=20)
    return out, model.log


def _run_native(stub, bodies):
    exe, tok_path = stub
    port = _free_port()
    proc = subprocess.Popen([exe, tok_path, str(port), str(len(bodies) + 1)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        _wait(port)
        out = [_post(port, b) for b in bodies]
    finally:
        try:
            log, _ = proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            log, _ = proc.communicate()
    return out, re.findall(r"POS \d+ \d+|CTL [^\n]*", log)   # the server's own log shares the lines


def _cell(**kw):
    return dict(kw, messages=MSGS)


VALID = [
    _cell(temperature=0, presence_penalty=1.5),
    _cell(temperature=0, frequency_penalty=2),
    _cell(temperature=0, logit_bias={"77": 100}),
    _cell(temperature=0, frequency_penalty=-0.5, presence_penalty=0.75, logit_bias={"5": -100, "300": 3.25, "0": 7}),
    _cell(temperature=0.8, seed=3, frequency_penalty=1.0, logit_bias={"12": 2.5}),
    _cell(temperature=0.8, seed=3, n=3, presence_penalty=-1.25, frequency_penalty=0.5, logit_bias={"5": -100, "9": 1e-3}),
    _cell(temperature=0, n=2, frequency_penalty=1.75, stream=True),
    _cell(temperature=1.3, top_p=0, seed=11, n=2, presence_penalty=2, stream=True, max_tokens=6),
    _cell(temperature=0.8, seed=3, n=3, max_tokens=5),
    _cell(temperature=0, max_tokens=5, logit_bias={str(i): -1.5 for i in range(100)}),
]


def test_servers_agree_on_controlled_completions(stub):
    py, py_log = _run_python(stub[1], VALID)
    nat, nat_log = _run_native(stub, VALID)
    for i, (a, b) in enumerate(zip(py, nat)):
        assert a and json.loads(a.split("data: ")[1] if a.startswith("data: ") else a) is not None
        # the servers escape non-ASCII text differently (test_api_completion_paths): compare parsed JSON pieces
        assert _parts(a) == _parts(b), i
    assert py_log == nat_log
    ctl = [ln for ln in py_log if ln.startswith("CTL ")]
    assert ctl[2] == "CTL 0 0 77:100" and ctl[3] == "CTL 0.75 -0.5 0:7 5:-100 300:3.25"
    # n = 3 sampled: every choice starts a completion of its own; greedy n = 2 runs once
    assert sum(1 for ln in ctl if ln.startswith("CTL -1.25 0.5 ")) == 3
    # the +100 bias wins every greedy draw until EOS
    j = json.loads(py[2])
    assert j["usage"]["completion_tokens"] == 13


def _parts(text: str):
    if not text.startswith("data: "):
        return json.loads(text)
    return [json.loads(p) if p != "[DONE]" else p for p in (x.strip() for x in text.split("data: ")) if p]


INVALID = [
    {"presence_penalty": 2.5}, {"presence_penalty": -2.01}, {"presence_penalty": "1"}, {"presence_penalty": None},
    {"presence_penalty": True}, {"frequency_penalty": 3}, {"frequency_penalty": [1]}, {"frequency_penalty": -1e300},
    {"logit_bias": []}, {"logit_bias": "x"}, {"logit_bias": None}, {"logit_bias": {"a": 1}}, {"logit_bias": {"-1": 1}},
    {"logit_bias": {"01": 1}}, {"logit_bias": {"1.0": 1}}, {"logit_bias": {" 1": 1}}, {"logit_bias": {"": 1}},
    {"logit_bias": {"99999999999": 1}}, {"logit_bias": {"1": 100.5}}, {"logit_bias": {"1": -101}}, {"logit_bias": {"1": "5"}},
    {"logit_bias": {"1": None}}, {"logit_bias": {str(i): 1 for i in range(101)}},
]


@pytest.mark.parametrize("server", ["python", "native"])
def test_invalid_controls_are_refused(stub, server):
    V = _H().Tokenizer(stub[1]).vocab_size
    bad = [_cell(temperature=0, **b) for b in INVALID] + [_cell(temperature=0, logit_bias={str(V): 1})]
    ok = _cell(temperature=0, max_tokens=3, presence_penalty=0.5)
    bodies = [x for b in bad for x in (b, ok)]
    out, log = (_run_python(stub[1], bodies) if server == "python" else _run_native(stub, bodies))
    for i in range(0, len(bodies), 2):
        assert out[i] == "", bodies[i]
        assert json.loads(out[i + 1])["usage"]["completion_tokens"] == 3, bodies[i]
    # a refused request reaches no backend: every prefill belongs to an answered request
    assert sum(1 for ln in log if ln.startswith("POS ")) == len(bad)
    # the highest valid id is accepted
    edge, _ = (_run_python if server == "python" else lambda s, b: _run_native(stub, b))(stub[1], [_cell(temperature=0, max_tokens=2, logit_bias={str(V - 1): 1})])
    assert json.loads(edge[0])["usage"]["completion_tokens"] == 2


@pytest.mark.parametrize("server", ["python", "native"])
def test_zero_controls_equal_no_controls(stub, server):
    base = [_cell(temperature=0), _cell(temperature=0.8, seed=5, n=3, max_tokens=6), _cell(temperature=1.0, seed=2, stream=True)]
    zero = [dict(b, presence_penalty=0, frequency_penalty=0.0, logit_bias={}) for b in base]
    run = _run_python if server == "python" else (lambda s, b: _run_native(stub, b))
    a, _ = run(stub[1], base)
    b, _ = run(stub[1], zero)
    assert a == b
