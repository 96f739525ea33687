"""`stop` strings on the real engine (tiny synthetic models): a completion ends at the token that completes the first occurrence of
a stop string and is cut right before it, on the single-sequence path of both servers and of InferenceSession, on the batched
choices step (`n` sampled), on the sequential choices of a mixture-of-experts model, under `--parallel 2`, and in streams."""
import http.client
import json
import os
import socket
import subprocess
import sys
import threading
import time

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MSGS = [{"role": "user", "content": "write something long"}]
# The tiny random models' plain greedy text repeats one byte that is not UTF-8; penalties keep a greedy completion varied.
VARIED = dict(presence_penalty=2.0, frequency_penalty=2.0)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class Server:
    def __init__(self, kind, model, parallel=1):
        m, t = model
        self.port = _free_port()
        cmd = ([sys.executable, "-m", "distributed_llama_b200.apps.api_server"] if kind == "python"
               else [os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")])
        self.proc = subprocess.Popen(cmd + ["--model", m, "--tokenizer", t, "--port", str(self.port), "--host", "127.0.0.1",
                                            "--temperature", "0", "--parallel", str(parallel)], cwd=ROOT,
                                     env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                     text=True, errors="replace")
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", self.port), timeout=0.5).close()
                return
            except OSError:
                assert self.proc.poll() is None, self.proc.stdout.read()
                time.sleep(0.2)

    def post(self, body):
        c = http.client.HTTPConnection("127.0.0.1", self.port, timeout=120)
        try:
            c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
            return c.getresponse().read()
        finally:
            c.close()

    def close(self):
        self.proc.kill()
        self.proc.communicate()


def _json(raw: bytes):
    return json.loads(raw.decode("utf-8", errors="replace"))


def _stream(raw: bytes, n=1):
    """(content per choice, chunks' contents per choice, log-probability entries per choice) of a stream."""
    content, chunks, entries = [""] * n, [[] for _ in range(n)], [[] for _ in range(n)]
    for line in raw.decode("utf-8", errors="replace").split("\r\n"):
        if not line.startswith("data: {"):
            continue
        c = json.loads(line[6:])["choices"][0]
        if "delta" in c:
            content[c["index"]] += c["delta"]["content"]
            chunks[c["index"]].append(c["delta"]["content"])
            entries[c["index"]] += c.get("logprobs", {}).get("content", [])
    return content, chunks, entries


def _pieces(entries):
    return [bytes(e["bytes"]) for e in entries]


def _stops(pieces):
    """Two stop strings from a greedy completion's token pieces: one that starts where a token's piece starts and one that
    starts inside a piece, each first occurring there, valid UTF-8 without replacement characters."""
    def ok(s: bytes, at: int) -> bool:
        try:
            t = s.decode("utf-8")
        except UnicodeDecodeError:
            return False
        return len(s) >= 2 and "�" not in t and b"".join(pieces).find(s) == at
    boundary = inside = None
    off = 0
    for k, p in enumerate(pieces):
        tail = b"".join(pieces[k:k + 3])
        if k >= 2 and boundary is None and ok(tail[:4], off):
            boundary = tail[:4].decode()
        for j in range(1, len(p)):
            if k >= 2 and inside is None and ok(tail[j:j + 4], off + j):
                inside = tail[j:j + 4].decode()
        off += len(p)
    assert boundary and inside, pieces
    return boundary, inside


def _ascii_stop(text):
    """Two printable ASCII characters of text (one if it has no such pair) from its third character on."""
    pairs = [text[i:i + 2] for i in range(2, len(text) - 1) if all(" " <= c <= "~" for c in text[i:i + 2])]
    singles = [c for c in text[2:] if " " <= c <= "~"]
    assert pairs or singles, text
    return pairs[0] if pairs else singles[0]


def _completing(pieces, stop: bytes):
    g = b""
    for k, p in enumerate(pieces):
        g += p
        if stop in g:
            return k
    return None


@pytest.mark.parametrize("kind", ["python", "native"])
def test_single_cut_and_stream(tmp_models, kind):
    """A single completion, greedy and sampled with a seed: cut at a stop string that starts where a token starts and at one
    that starts inside a token's piece."""
    srv = Server(kind, tmp_models["tiny-llama31"])
    try:
        for sampling in (dict(temperature=0, **VARIED), dict(temperature=0.9, seed=23)):
            base = dict(messages=MSGS, max_tokens=48, logprobs=True, top_logprobs=2, **sampling)
            plain = _json(srv.post(base))
            text = plain["choices"][0]["message"]["content"]
            entries = plain["choices"][0]["logprobs"]["content"]
            pieces = _pieces(entries)
            for stop in _stops(pieces):
                k = _completing(pieces, stop.encode())
                got = _json(srv.post(dict(base, stop=stop)))
                content = got["choices"][0]["message"]["content"]
                assert content == text[:text.find(stop)], stop
                assert got["usage"]["completion_tokens"] == k + 1
                assert got["choices"][0]["logprobs"]["content"] == entries[:k + 1]
                # the stream: the same content and entries, and no chunk reaches past the cut
                s_content, chunks, s_entries = _stream(srv.post(dict(base, stop=[stop], stream=True)))
                assert s_content[0] == content and s_entries[0] == entries[:k + 1]
                seen = ""
                for c in chunks[0]:
                    seen += c
                    assert content.startswith(seen)
        # n = 3 sampled with a seed (batched choices step): each choice is its own run cut at its own first occurrence
        body = dict(messages=MSGS, max_tokens=32, n=3, temperature=0.9, seed=17)
        runs = [c["message"]["content"] for c in _json(srv.post(body))["choices"]]
        stop = _ascii_stop(runs[0])
        cut = [c["message"]["content"] for c in _json(srv.post(dict(body, stop=stop)))["choices"]]
        assert any(stop in r for r in runs)
        for r, c in zip(runs, cut):
            assert c == (r[:r.find(stop)] if stop in r else r)
        s_content, _, _ = _stream(srv.post(dict(body, stop=stop, stream=True)), 3)
        assert s_content == cut
    finally:
        srv.close()


@pytest.mark.parametrize("kind", ["python", "native"])
def test_parallel_slots(tmp_models, kind):
    """--parallel 2: a request with `stop` next to one without; the latter returns what it returns alone."""
    srv = Server(kind, tmp_models["tiny-llama31"], parallel=2)
    try:
        a = dict(messages=MSGS, max_tokens=48, logprobs=True, **VARIED)
        b = dict(messages=[{"role": "user", "content": "another prompt"}], max_tokens=48)
        plain_a = _json(srv.post(a))["choices"][0]
        alone_b = _json(srv.post(b))["choices"][0]["message"]["content"]
        stop = _stops(_pieces(plain_a["logprobs"]["content"]))[0]
        text = plain_a["message"]["content"]
        out = [None, None]

        def go(i, body):
            out[i] = _json(srv.post(body))["choices"][0]["message"]["content"]
        ths = [threading.Thread(target=go, args=(0, dict(a, stop=stop))), threading.Thread(target=go, args=(1, b))]
        for t in ths:
            t.start()
        for t in ths:
            t.join(timeout=120)
        assert out[0] == text[:text.find(stop)] and out[1] == alone_b
    finally:
        srv.close()


def test_session_and_sequential_choices(tmp_models):
    """InferenceSession.generate_choices: greedy on a dense model, and sampled n = 3 on a mixture-of-experts model (the
    choices run one after another)."""
    from distributed_llama_b200.api import InferenceSession
    for name, T in (("tiny-llama31", 0.0), ("tiny-qwen3-moe", 0.9)):
        m, t = tmp_models[name]
        runs = InferenceSession(m, t, temperature=T, seed=3, **VARIED).generate_choices("hello world", 3, 32, seed=11)
        stop = _ascii_stop(runs[0])
        cut = InferenceSession(m, t, temperature=T, seed=3, **VARIED).generate_choices("hello world", 3, 32, seed=11, stop=[stop])
        for r, c in zip(runs, cut):
            assert c == (r[:r.find(stop)] if stop in r else r), (name, stop)
        assert any(stop in r for r in runs)
