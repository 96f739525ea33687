"""`stop` strings without a GPU: the host StopMatcher against a plain Python model of the rule, the `stop` field's parsing and
refusals, and both chat servers over stub models (tests/native/api_stop_stub_main.cpp and its twin StopStub, and the --parallel
stub of tests/test_api_parallel.py): the same responses from both, the cut, the stream's hold-back, log-probability entries,
the prompt cache after a cut, and a cut request freeing its slot for a waiting one."""
import json
import os
import random
import re
import socket
import subprocess
import threading
import time
from types import SimpleNamespace

import pytest

from distributed_llama_b200 import host
from distributed_llama_b200.api import check_stop
from distributed_llama_b200.apps.api_server import parse_stop
import test_sampling_controls as tsc  # its raw-socket client and parsed-response helpers
from test_logprobs_args import LogprobsStub
from test_api_parallel import SlotStub, _concurrent, _msgs
from test_api_parallel import _post as _post_contents

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the matcher ---------------------------------------------------------------------------------------------------------------

def model(stops, deltas):
    """The rule on the whole text G: after each delta, the first occurrence of any stop string ends the text at its start; else
    every byte of G except its longest suffix that is a proper prefix of some stop string can no longer be cut. Returns the
    bytes released per delta, the index of the delta that matched (None) and the bytes still held at the end."""
    G, sent, out = b"", 0, []
    for k, d in enumerate(deltas):
        G += d
        starts = [G.find(s) for s in stops if s in G]
        if starts:
            out.append(G[sent:min(starts)])
            return out, k, b""
        hold = max((n for s in stops for n in range(1, len(s)) if G.endswith(s[:n])), default=0)
        assert len(G) - hold >= sent
        out.append(G[sent:len(G) - hold])
        sent = len(G) - hold
    return out, None, G[sent:]


def run_matcher(stops, deltas):
    m = host().StopMatcher(stops)
    out, hit = [], None
    for k, d in enumerate(deltas):
        out.append(m.push(d))
        if m.stopped:
            hit = k
            break
    return out, hit, m.flush()


STREAMS = {
    "inside one piece": ([b"lo"], [b"Hel", b"xloy", b"z"]),
    "across three pieces": ([b"STOP"], [b"ab S", b"T", b"OP tail", b"more"]),
    "prefix of another": ([b"abc", b"ab"], [b"xa", b"bc", b"d"]),
    "prefix of another, longer first in the text": ([b"ab", b"abX"], [b"a", b"bX"]),
    "later start completes first": ([b"abcd", b"bc"], [b"a", b"b", b"c", b"d"]),
    "hold back then release": ([b"END"], [b"xE", b"N", b"x", b"y"]),
    "hold back released at the end": ([b"END"], [b"xE", b"N"]),
    "two-byte character split": (["é".encode()], [b"ab\xc3", b"\xa9cd"]),
    "four-byte character split": (["😀".encode()], [b"x\xf0\x9f", b"\x98", b"\x80y"]),
    "equal to a whole piece": ([b" world"], [b"Hello", b" world", b"!"]),
    "first delta": ([b"He"], [b"Hello", b" there"]),
    "empty deltas": ([b"ab"], [b"", b"a", b"", b"b"]),
    "no stop strings": ([], [b"Hello", b" world", b"\xc3\xa9"]),
}


@pytest.mark.parametrize("name", sorted(STREAMS))
def test_matcher_follows_the_rule(name):
    stops, deltas = STREAMS[name]
    assert run_matcher(stops, deltas) == model(stops, deltas)


def test_matcher_cuts():
    assert b"".join(run_matcher([b"lo"], [b"Hel", b"xloy", b"z"])[0]) == b"Helx"
    assert run_matcher([b"STOP"], [b"ab S", b"T", b"OP tail"])[:2] == ([b"ab ", b"", b""], 2)
    assert b"".join(run_matcher([b"abcd", b"bc"], [b"a", b"b", b"c", b"d"])[0]) == b"a"
    assert run_matcher([b"END"], [b"xE", b"N", b"x"])[0] == [b"x", b"", b"ENx"]
    assert run_matcher([b"He"], [b"Hello"])[:2] == ([b""], 0)
    assert run_matcher([], [b"Hello", b" world"]) == ([b"Hello", b" world"], None, b"")


def test_matcher_random_streams():
    rs = random.Random(7)
    for _ in range(3000):
        stops = [bytes(rs.choice(b"abc") for _ in range(rs.randint(1, 5))) for _ in range(rs.randint(1, 4))]
        deltas = [bytes(rs.choice(b"abcd") for _ in range(rs.randint(0, 4))) for _ in range(rs.randint(1, 8))]
        assert run_matcher(stops, deltas) == model(stops, deltas), (stops, deltas)


def test_matcher_refuses_an_empty_stop_string():
    with pytest.raises(ValueError):
        host().StopMatcher([b"a", b""])


# ---- the `stop` field ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("stop,want", [(None, []), ([], []), ("x", [b"x"]), (["a", "bc"], [b"a", b"bc"]), ("é", ["é".encode()]),
                                       (["a", "b", "c", "d"], [b"a", b"b", b"c", b"d"]), ("x" * 256, [b"x" * 256]),
                                       ("😀", ["😀".encode()])])
def test_parse_accepts(stop, want):
    assert check_stop(stop) == want
    assert parse_stop({"stop": stop}) == want
    assert parse_stop({}) == []


BAD_STOP = [1, 1.5, True, {"a": "b"}, [1], ["a", 2], ["a", None], "", [""], ["a"] * 5, "x" * 257, "é" * 129, "\ud800", "a\udc00",
            ["ok", "\ud83d"], [["a"]]]


@pytest.mark.parametrize("stop", BAD_STOP, ids=range(len(BAD_STOP)))
def test_parse_refuses(stop):
    with pytest.raises(ValueError):
        parse_stop({"stop": stop})


# ---- both servers over a stub model ----------------------------------------------------------------------------------------------

def _compile(tmp_path_factory, name, main):
    d = str(tmp_path_factory.mktemp(name))
    exe = os.path.join(d, name)
    srcs = [os.path.join(ROOT, "tests", "native", main), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe, "-lpthread"], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


@pytest.fixture(scope="module")
def stop_stub(tmp_path_factory):
    return _compile(tmp_path_factory, "api_stop_stub", "api_stop_stub_main.cpp")


@pytest.fixture(scope="module")
def parallel_stub(tmp_path_factory):
    return _compile(tmp_path_factory, "api_parallel_stub", "api_parallel_stub_main.cpp")


class StopStub(LogprobsStub):
    """tests/native/api_stop_stub_main.cpp in Python: LogprobsStub that logs every prefill as (start, n)."""

    def __init__(self, V, eos):
        super().__init__(V, eos)
        self.prefills = []

    def prefill(self, tokens, pos):
        self.prefills.append((pos, len(tokens)))
        super().prefill(tokens, pos)


class Servers:
    """The Python server over StopStub and the native stub, sent the same requests in the same order. `budget` bounds the
    requests; close() uses up the rest with bodies both refuse, so that both servers end."""

    def __init__(self, stub, budget=40):
        from distributed_llama_b200.apps import api_server as py_api
        from distributed_llama_b200.apps.args import parse_args
        exe, tok_path = stub
        H = host()
        tok = H.Tokenizer(tok_path)
        self.model = StopStub(tok.vocab_size, list(tok.eos_ids)[0])
        self.py_port, self.nat_port, self.left = tsc._free_port(), tsc._free_port(), budget
        args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(self.py_port),
                           "--temperature", "0"], False)
        ctx = SimpleNamespace(args=args, sess=None, inference=self.model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                              header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
        self.thread = threading.Thread(target=py_api.serve, args=(ctx, budget + 1), daemon=True)
        self.thread.start()
        self.proc = subprocess.Popen([exe, tok_path, str(self.nat_port), str(budget + 1)], stdout=subprocess.PIPE,
                                     stderr=subprocess.STDOUT, text=True, errors="replace")
        tsc._wait(self.py_port)
        tsc._wait(self.nat_port)

    def post(self, body):
        """(Python response, native response), each without its `created` stamps ("" when refused)."""
        assert self.left > 0
        self.left -= 1
        return tsc._post(self.py_port, body), tsc._post(self.nat_port, body)

    def follow_up(self, answers, messages):
        """The follow-up of `messages` that quotes each server's own answer (post's results), then asks for more."""
        assert self.left > 0
        self.left -= 1
        tsc._post(self.py_port, _follow_up(answers[0], messages))
        tsc._post(self.nat_port, _follow_up(answers[1], messages))

    def close(self):
        """Native prefill log as (start, n) pairs."""
        while self.left > 0:
            self.post(b"{")
        self.thread.join(timeout=20)
        try:
            log, _ = self.proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            log, _ = self.proc.communicate()
        return [(int(a), int(b)) for a, b in re.findall(r"POS (\d+) (\d+)\n", log)]


MSGS = [{"role": "user", "content": "hello"}]


def _follow_up(response: str, messages) -> bytes:
    """A body that extends `messages` with the assistant content of a non-stream response, quoted as the bytes the server wrote
    (the native server passes the decoder's bytes through, the Python server writes them as decoded with replacement), and a
    user turn."""
    raw = response.encode("utf-8", "surrogateescape")
    lit = re.search(rb'"content": ("(?:[^"\\]|\\.)*")', raw).group(1)
    body = json.dumps(dict(messages=messages + [{"role": "assistant", "content": "@@"}, {"role": "user", "content": "more"}]))
    return body.encode().replace(b'"@@"', lit)


def _content(text, i=0):
    """Choice i's content of a JSON body or a stream (its deltas joined)."""
    parts = tsc._parts(text)
    if isinstance(parts, dict):
        return parts["choices"][i]["message"]["content"]
    return "".join(p["choices"][0]["delta"]["content"] for p in parts
                   if isinstance(p, dict) and p["choices"][0]["index"] == i and "delta" in p["choices"][0])


def _ascii_runs(text, n):
    """Every n-character run of printable ASCII in text, with its first index."""
    return [(text[k:k + n], k) for k in range(len(text) - n + 1) if all(" " <= c <= "~" for c in text[k:k + n])]


def _pick(text, n, after=0):
    """A printable ASCII string of n characters whose first occurrence in text lies at `after` or later."""
    for s, k in _ascii_runs(text, n):
        if k >= after and text.find(s) == k:
            return s, k
    raise AssertionError(f"no ASCII run of {n} in {text!r}")


def _completing_token(entries, stop: bytes):
    """Index of the token whose bytes complete the first occurrence of stop (log-probability entries' `bytes`)."""
    g = b""
    for k, e in enumerate(entries):
        g += bytes(e["bytes"])
        if stop in g:
            return k
    return None


def test_servers_agree_and_cut(stop_stub):
    srv = Servers(stop_stub)
    try:
        base = dict(messages=MSGS, logprobs=True, top_logprobs=2)
        py, nat = srv.post(base)
        assert tsc._parts(py) == tsc._parts(nat)
        full = json.loads(py)
        text, entries = full["choices"][0]["message"]["content"], full["choices"][0]["logprobs"]["content"]
        s1, k1 = _pick(text, 2, after=3)
        s2, k2 = _pick(text, 3, after=k1 + 3) if len(text) > k1 + 6 else (s1, k1)
        never = "~~never~~"
        assert never not in text
        first = text[0]
        cases = [(dict(base, stop=s1), s1), (dict(base, stop=[never, s2, s1]), s1), (dict(base, stop=[s2]), s2),
                 (dict(base, stop=first), first)]
        for body, s in cases:
            for stream in (False, True):
                py, nat = srv.post(dict(body, stream=stream))
                assert py and tsc._parts(py) == tsc._parts(nat), body
                assert _content(py) == text[:text.find(s)], body
                if not stream:
                    j = json.loads(py)
                    k = _completing_token(entries, s.encode())
                    # the token that completed the match counts and has its entry, whose bytes reach past the content
                    assert j["usage"]["completion_tokens"] == k + 1
                    assert j["choices"][0]["logprobs"]["content"] == entries[:k + 1]
                else:
                    parts = tsc._parts(py)
                    lp = [e for p in parts if isinstance(p, dict) for e in p["choices"][0].get("logprobs", {}).get("content", [])]
                    assert lp == entries[:_completing_token(entries, s.encode()) + 1]
                    assert parts[-2]["choices"][0]["finish_reason"] == "stop" and parts[-1] == "[DONE]"
        # a stop string never reached: the same response as without the field, stream and not
        for stream in (False, True):
            with_stop, _ = srv.post(dict(base, stop=[never], stream=stream))
            without, _ = srv.post(dict(base, stream=stream))
            assert with_stop == without
        # n = 3 sampled with a seed: each choice is cut at its own first occurrence, the others are unchanged
        body = dict(messages=MSGS, n=3, temperature=0.8, seed=5)
        py, _ = srv.post(body)
        plain = [c["message"]["content"] for c in json.loads(py)["choices"]]
        s, _ = _pick(plain[0], 2, after=2)
        for stream in (False, True):
            py, nat = srv.post(dict(body, stop=s, stream=stream))
            assert tsc._parts(py) == tsc._parts(nat)
            for i in range(3):
                want = plain[i][:plain[i].find(s)] if s in plain[i] else plain[i]
                assert _content(py, i) == want, i
    finally:
        srv.close()


def test_stream_holds_back_partial_matches(stop_stub):
    """No stream chunk carries a byte past the cut, and a partial match released later arrives whole."""
    srv = Servers(stop_stub)
    try:
        py, _ = srv.post(dict(messages=MSGS))
        text = _content(py)
        s, k = _pick(text, 3, after=2)
        # a stop string whose first two characters occur in the text but whose end does not: held back, then released
        partial = s[:2] + "\x7f"
        assert partial not in text
        for stop in ([s], [partial], [partial, s]):
            py, nat = srv.post(dict(messages=MSGS, stream=True, stop=stop))
            assert tsc._parts(py) == tsc._parts(nat)
            got = [p["choices"][0]["delta"]["content"] for p in tsc._parts(py) if isinstance(p, dict) and "delta" in p["choices"][0]]
            want = text[:text.find(s)] if s in stop else text
            assert "".join(got) == want
            seen = ""
            for g in got:
                seen += g
                assert want.startswith(seen)
    finally:
        srv.close()


BAD_BODIES = [dict(messages=MSGS, stop=s) for s in BAD_STOP]


@pytest.mark.parametrize("server", ["python", "native"])
def test_malformed_stop_is_refused(stop_stub, server):
    srv = Servers(stop_stub, budget=2 * len(BAD_BODIES) + 2)
    try:
        ok = dict(messages=MSGS, max_tokens=3, stop=["~~never~~"])
        for bad in BAD_BODIES:
            py, nat = srv.post(bad)
            assert (py if server == "python" else nat) == "", bad
            py, nat = srv.post(ok)
            assert json.loads(py if server == "python" else nat)["usage"]["completion_tokens"] == 3
        # an escaped unpaired surrogate written by hand, and a valid pair next to it
        raw = b'{"messages": [{"role": "user", "content": "hello"}], "max_tokens": 2, "stop": ["\\ud800\\u0041"]}'
        py, nat = srv.post(raw)
        assert (py if server == "python" else nat) == ""
        py, nat = srv.post(raw.replace(b"\\u0041", b"\\udc00"))
        assert json.loads(py if server == "python" else nat)["usage"]["completion_tokens"] == 2
    finally:
        srv.close()


def test_prompt_cache_after_a_cut(stop_stub):
    srv = Servers(stop_stub)
    try:
        a = [{"role": "user", "content": "first question"}]
        b = [{"role": "user", "content": "second question"}]
        probe, _ = srv.post(dict(messages=a))
        text = _content(probe)
        s, _ = _pick(text, 2, after=2)
        # a cut answer: the cache ends at the prompt, and the follow-up quoting the answer prefills it from there
        cut = srv.post(dict(messages=a, stop=s))
        assert tsc._parts(cut[0]) == tsc._parts(cut[1])
        n_prompt = json.loads(cut[0])["usage"]["prompt_tokens"]
        srv.follow_up(cut, a)
        # the same body without a match still caches its answer: its follow-up starts after the answer
        whole = srv.post(dict(messages=b, stop="~~never~~"))
        usage = json.loads(whole[0])["usage"]
        srv.follow_up(whole, b)
    finally:
        nat_pos = srv.close()
    py_pos = srv.model.prefills
    assert py_pos == nat_pos
    # probe, cut, follow-up of the cut, uncut, follow-up of the uncut
    assert [p[0] for p in py_pos] == [0, 0, n_prompt - 1, 0, usage["prompt_tokens"] - 1 + usage["completion_tokens"]]


# ---- --parallel -------------------------------------------------------------------------------------------------------------------

class ParallelServers:
    """The Python --parallel server over SlotStub and the native --parallel stub."""

    def __init__(self, stub, budget, parallel=2, eos_after=10, delay_ms=20):
        from distributed_llama_b200.apps import api_server as py_api
        from distributed_llama_b200.apps.args import parse_args
        exe, tok_path = stub
        H = host()
        tok = H.Tokenizer(tok_path)
        self.model = SlotStub(parallel, 1024 // parallel, tok.regular_vocab_size, list(tok.eos_ids)[0], eos_after, delay_ms / 1000)
        self.py_port, self.nat_port = tsc._free_port(), tsc._free_port()
        args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(self.py_port),
                           "--temperature", "0", "--parallel", str(parallel)], False)
        ctx = SimpleNamespace(args=args, sess=None, inference=self.model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 77),
                              header=SimpleNamespace(seq_len=1024, vocab_size=tok.vocab_size))
        self.thread = threading.Thread(target=py_api.serve, args=(ctx, budget + 1), daemon=True)
        self.thread.start()
        self.proc = subprocess.Popen([exe, tok_path, str(self.nat_port), str(budget + 1), str(parallel), str(eos_after), str(delay_ms)],
                                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, errors="replace")
        tsc._wait(self.py_port)
        tsc._wait(self.nat_port)

    def close(self):
        self.thread.join(timeout=30)
        try:
            log, _ = self.proc.communicate(timeout=30)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            log, _ = self.proc.communicate()
        return [tuple(int(x) for x in m) for m in re.findall(r"POS (\d+) (\d+) (\d+)\n", log)]


def _ascii_stop(text, after):
    for s, k in _ascii_runs(text, 1):
        if k >= after and text.find(s) == k:
            return s
    raise AssertionError(f"no ASCII character in {text!r}")


def test_parallel_servers_agree_and_keep_the_cache_at_the_prompt(parallel_stub):
    srv = ParallelServers(parallel_stub, budget=7)
    try:
        def both(body, nat_body=None):
            return tsc._post(srv.py_port, body), tsc._post(srv.nat_port, body if nat_body is None else nat_body)
        plain, _ = both(dict(messages=_msgs(0)))
        text = _content(plain)
        s = _ascii_stop(text, 1)
        cut = both(dict(messages=_msgs(0), stop=s))
        assert tsc._parts(cut[0]) == tsc._parts(cut[1]) and _content(cut[0]) == text[:text.find(s)]
        streamed = both(dict(messages=_msgs(0), stop=s, stream=True))
        assert tsc._parts(streamed[0]) == tsc._parts(streamed[1]) and _content(streamed[0]) == text[:text.find(s)]
        n_prompt = json.loads(cut[0])["usage"]["prompt_tokens"]
        both(*(_follow_up(c, _msgs(0)) for c in cut))
        sampled = both(dict(messages=_msgs(1), n=2, temperature=0.8, seed=9, stop=s))
        assert tsc._parts(sampled[0]) == tsc._parts(sampled[1])
        uncut = both(dict(messages=_msgs(2), stop="~~never~~"))
        usage = json.loads(uncut[0])["usage"]
        both(*(_follow_up(c, _msgs(2)) for c in uncut))
    finally:
        nat_pos = srv.close()
    assert srv.model.prefills == nat_pos
    starts = [p[1] for p in nat_pos]
    # plain, cut, streamed cut, its follow-up from the prompt end, n = 2, uncut, its follow-up after the answer
    assert starts[3] == n_prompt - 1
    assert starts[-1] == usage["prompt_tokens"] - 1 + usage["completion_tokens"]


def test_parallel_cut_frees_its_slot(parallel_stub):
    """Two slots, three long requests: the first ends at a stop string early, so the third starts before the second ends. The
    request without `stop` returns what it returns alone."""
    srv = ParallelServers(parallel_stub, budget=6, eos_after=30, delay_ms=30)
    try:
        for port in (srv.py_port, srv.nat_port):
            a, b = dict(messages=_msgs(0), stream=True), dict(messages=_msgs(1), stream=True)
            text = _post_contents(port, a)[0]
            alone_b = _post_contents(port, b)
            s = _ascii_stop(text, 2)
            out, stamps = _concurrent(port, [dict(a, stop=s), b, dict(messages=_msgs(2), stream=True)], stagger=0.01)
            assert out[0] == [text[:text.find(s)]] and out[1] == alone_b and len(out[2][0]) > 0, port
            assert stamps[2][0] < stamps[1][-1], port       # the waiting request started before the long one ended
    finally:
        srv.close()
