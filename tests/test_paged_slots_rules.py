"""Paged KV-cache slots on the CPU: `--parallel-cache` parsing and refusals in both servers, and SlotScheduler's pool rules over a
stub backend that keeps pages the way the engine does (csrc/cuda/engine.cu: dl_engine_slot_reserve, lowest free page first)."""
import os
import subprocess
import threading

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = 64


class PagedStub:
    """`slots` slots over a pool of `pages` 64-row pages. A row's next token depends on (token, position) only; a step that writes
    a row outside its slot's pages fails the test."""
    paged = True

    def __init__(self, slots, pages):
        self.slots, self.slot_len = slots, pages * PAGE
        self.table = [[] for _ in range(slots)]
        self.used = [False] * pages
        self.log = []

    def slot_reserve(self, slot, rows):
        need = -(-rows // PAGE) - len(self.table[slot])
        free = [p for p, u in enumerate(self.used) if not u]
        if need <= 0:
            return True
        if len(free) < need:
            return False
        for p in free[:need]:
            self.used[p] = True
            self.table[slot].append(p)
        return True

    def slot_trim(self, slot, rows):
        t = self.table[slot]
        while len(t) > -(-rows // PAGE):
            self.used[t.pop()] = False

    def slot_release(self, slot):
        self.slot_trim(slot, 0)
        self.log.append(("release", slot))

    def free_pages(self):
        return self.used.count(False)

    def slot_pages(self, slot):
        return list(self.table[slot])

    def slot_prefill(self, slot, tokens, pos):
        assert pos + len(tokens) <= len(self.table[slot]) * PAGE
        self.log.append(("prefill", slot, pos, len(tokens)))

    def slot_copy(self, src, dst, P):
        assert self.slot_reserve(dst, P)

    def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias, **filters):
        pass

    def slots_step(self, tokens, pos, active):
        for b in range(self.slots):
            if active[b]:
                assert pos[b] < len(self.table[b]) * PAGE, (b, pos[b], self.table[b])
        return [(t * 7 + p * 13 + 5) % 500 + 1 if a else -1 for t, p, a in zip(tokens, pos, active)]


class Req:
    """A greedy request over a token prompt; the slot's prompt cache is a token prefix (`caches`, shared by the requests)."""

    def __init__(self, log, name, prompt, max_tokens, caches, n=1, temperature=0.0):
        from distributed_llama_b200.api import SlotRequest
        self.__class__ = type("R", (Req, SlotRequest), {})
        self.log, self.name, self.prompt, self.max_tokens, self.caches = log, name, prompt, max_tokens, caches
        self.n, self.temperature, self.seed = n, temperature, 1
        self.out, self.error, self.done = None, None, threading.Event()

    def cached_prefix(self, slot):
        c = self.caches[slot]
        return len(c) if c and len(c) < len(self.prompt) and self.prompt[:len(c)] == c else 0

    def prompt_len(self, slot):
        return len(self.prompt) - 1

    def prepare(self, slot):
        start = self.cached_prefix(slot)
        self.log.append(("admit", self.name, slot, start))
        self.caches[slot] = list(self.prompt)
        return self.prompt[start:-1], start, self.prompt[-1], len(self.prompt) - 1

    def on_token(self, i, tok):
        return False

    def finish(self, out, slots, P):
        self.caches[slots[0]] = self.prompt + out[0][:-1]
        self.out = out
        self.log.append(("finish", self.name))
        self.done.set()

    def fail(self, e, slots):
        self.error = e
        self.log.append(("fail", self.name))
        self.done.set()


def _run(stub, caches, batches):
    """Serves the batches of requests in turn, a batch (or a function returning one) once the previous one is done; returns the
    evicted slots."""
    from distributed_llama_b200.api import SlotScheduler
    evicted = []

    def on_evict(s):
        evicted.append(s)
        caches[s] = None

    sched = SlotScheduler(stub, lambda: 1, on_evict=on_evict)
    t = threading.Thread(target=sched.run, daemon=True)
    t.start()
    for batch in batches:
        batch = batch() if callable(batch) else batch   # built once the batches before it are done
        for r in batch:
            sched.submit(r)
        for r in batch:
            assert r.done.wait(30), r.name
    sched.stop()
    t.join(10)
    return evicted


def _prompt(n, salt):
    return [(7 * i + salt) % 500 + 1 for i in range(n)]


def test_admission_evicts_idle_caches_least_recently_finished_first():
    stub, log, caches = PagedStub(3, 6), [], [None] * 3
    # slots 0, 1, 2; 2 pages each (rows [0, 19 + 64)); they finish in the order z, y, x
    y, x, z = (Req(log, n, _prompt(20, k), m, caches) for n, k, m in (("y", 1, 10), ("x", 2, 30), ("z", 3, 5)))
    a = Req(log, "a", _prompt(200, 4), 10, caches)          # P = 199: rows [0, 263) = 5 pages; takes slot 0 (y's 2 pages)
    later = []

    def follow_up():
        later.append(Req(log, "x2", x.prompt + x.out[0] + [9], 3, caches))
        return later
    assert _run(stub, caches, [[y, x, z], [a], follow_up]) == [2, 1]   # z's cache, then x's
    assert [e[1:3] for e in log if e[0] == "admit"][:3] == [("y", 0), ("x", 1), ("z", 2)]
    assert [e[1] for e in log if e[0] == "finish"][:3] == ["z", "y", "x"]
    assert [e for e in log if e[:2] == ("admit", "x2")][0][3] == 0   # x's prefix is gone with its cache


def test_blocked_admission_is_first_in_first_out():
    stub, log, caches = PagedStub(2, 4), [], [None] * 2
    a = Req(log, "a", _prompt(130, 1), 20, caches)          # needs the whole pool
    b = Req(log, "b", _prompt(10, 2), 5, caches)
    _run(stub, caches, [[a, b]])
    admits = [i for i, e in enumerate(log) if e[0] == "admit"]
    assert log[admits[0]][1] == "a"
    assert log.index(("finish", "a")) < admits[1]          # b waited although a slot was free


def test_row_without_a_page_ends_with_a_prefix_of_its_solo_run():
    stub, log, caches = PagedStub(2, 4), [], [None] * 2
    c, d = Req(log, "c", _prompt(20, 3), 230, caches), Req(log, "d", _prompt(20, 6), 230, caches)
    _run(stub, caches, [[c, d]])
    lens = sorted(len(r.out[0]) for r in (c, d))
    assert lens[0] < 230 and lens[1] == 230
    cut = c if len(c.out[0]) < 230 else d
    assert len(cut.out[0]) == 128 - 19                      # rows 19 .. 127: the two pages it had
    solo_stub, solo_caches = PagedStub(2, 4), [None] * 2
    solo = Req([], "solo", cut.prompt, 230, solo_caches)
    _run(solo_stub, solo_caches, [[solo]])
    assert solo.out[0][:len(cut.out[0])] == cut.out[0]


def test_request_larger_than_the_pool_fails():
    stub, log, caches = PagedStub(4, 4), [], [None] * 4
    r = Req(log, "r", _prompt(100, 1), 5, caches, n=3, temperature=0.7)   # 3 slots x 3 pages > 4
    _run(stub, caches, [[r]])
    assert r.error is not None and "pages" in str(r.error)


def test_hook_error_reaches_fail_as_the_same_object():
    """An exception a request's hook raises reaches its fail as the same object and frees its pages, while the other request
    finishes; the scheduler's own refusal of a request arrives as ValueError."""
    stub, log, caches = PagedStub(3, 6), [], [None] * 3
    gone = ConnectionError("the client went away")
    a, b = Req(log, "a", _prompt(20, 1), 10, caches), Req(log, "b", _prompt(20, 2), 10, caches)
    wide = Req(log, "wide", _prompt(20, 3), 5, caches, n=4, temperature=0.7)   # 4 completions, 3 slots
    none = Req(log, "none", _prompt(20, 4), 5, caches, n=0)

    def on_token(i, tok):
        raise gone
    a.on_token = on_token
    _run(stub, caches, [[a, b, wide, none]])
    assert a.error is gone and a.out is None
    slot = [e for e in log if e[:2] == ("admit", "a")][0][2]
    assert ("release", slot) in stub.log                       # a's slot gives its pages back
    assert b.error is None and len(b.out[0]) == 10
    assert type(wide.error) is ValueError and str(wide.error) == "n = 4 needs more than the 3 slots"
    assert type(none.error) is ValueError and str(none.error) == "n must be at least 1"


def test_seeds_are_taken_modulo_2_64():
    """A request's seed reaches the slots as the engine takes it, modulo 2^64: itself for one completion, choice_seed of it for
    several, so a negative seed serves n > 1 too."""
    from distributed_llama_b200 import host

    class SeedStub(PagedStub):
        def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias, **filters):
            self.log.append(("seed", slot, seed))

    stub, log, caches = SeedStub(3, 6), [], [None] * 3
    one, two = Req(log, "one", _prompt(20, 1), 3, caches, temperature=0.7), Req(log, "two", _prompt(20, 2), 3, caches, n=2, temperature=0.7)
    one.seed = two.seed = -5
    _run(stub, caches, [[one], [two]])
    assert one.error is None and two.error is None
    seeds = [e[2] for e in stub.log if e[0] == "seed"]
    assert seeds == [2**64 - 5] + [host().choice_seed(2**64 - 5, i) for i in range(2)]


def test_idle_run_stops_on_sigint():
    """run() on the main thread with nothing to do raises KeyboardInterrupt on Ctrl-C, without waiting for a request."""
    import signal
    import time
    from distributed_llama_b200.api import SlotScheduler
    sched = SlotScheduler(PagedStub(2, 4), lambda: 1)
    old = signal.signal(signal.SIGINT, signal.default_int_handler)
    interrupt = threading.Timer(0.3, lambda: os.kill(os.getpid(), signal.SIGINT))
    watchdog = threading.Timer(10, sched.stop)   # a run() that misses the signal returns here, too late
    try:
        interrupt.start()
        watchdog.start()
        t0 = time.monotonic()
        with pytest.raises(KeyboardInterrupt):
            sched.run()
        assert time.monotonic() - t0 < 5
    finally:
        interrupt.cancel()
        watchdog.cancel()
        signal.signal(signal.SIGINT, old)


def test_pages_are_taken_lowest_first():
    stub = PagedStub(2, 6)
    assert stub.slot_reserve(0, 65) and stub.slot_reserve(1, 1)
    stub.slot_release(0)
    assert stub.slot_reserve(1, 130) and stub.table[1] == [2, 0, 1]
    assert not stub.slot_reserve(0, 4 * PAGE) and stub.table[0] == []


# ---- --parallel-cache in both servers ---------------------------------------------------------------------------------------------

def test_parallel_cache_parsing():
    from distributed_llama_b200.api import parallel_refusal
    from distributed_llama_b200.apps.args import parse_args
    assert parse_args(["--model", "m", "--parallel-cache", "paged"], False).parallel_cache == "paged"
    assert parse_args(["--model", "m"], False).parallel_cache == "split"
    assert parallel_refusal(4, 1, 0, "paged") is None and parallel_refusal(4, 1, 0, "split") is None
    assert "--parallel-cache" in parallel_refusal(4, 1, 0, "pages")
    assert "mixture-of-experts" in parallel_refusal(4, 1, 8, "paged")   # the other refusals apply unchanged
    assert "one GPU" in parallel_refusal(4, 2, 0, "paged")


def test_python_server_refuses_unknown_layout(capsys):
    from distributed_llama_b200.apps import api_server as py_api
    assert py_api.main(["--model", "m.m", "--tokenizer", "t.t", "--parallel", "2", "--parallel-cache", "bogus"]) == 1
    err = capsys.readouterr().err.strip()
    assert "--parallel-cache" in err and len(err.splitlines()) == 1


@pytest.mark.parametrize("value", ["bogus", "pages"])
def test_native_server_refuses(value):
    """An unknown layout is refused in one line."""
    exe = os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")
    if not os.path.exists(exe):
        from distributed_llama_b200 import _build
        _build.build_all(verbose=False)
    env = {k: v for k, v in os.environ.items() if k not in ("DL_COLLECTIVES", "DL_HOST_SAMPLER")}
    r = subprocess.run([exe, "--model", "m.m", "--tokenizer", "t.t", "--parallel", "2", "--parallel-cache", value], capture_output=True,
                       text=True, env=env, timeout=30)
    assert r.returncode == 1
    assert "--parallel-cache" in r.stderr and len(r.stderr.strip().splitlines()) == 1


def test_a_slot_taken_gives_back_the_pages_it_does_not_need():
    """A long finished conversation's slot is taken by a short request: the pages past what that request needs go back to the pool,
    so a second short request runs beside it instead of waiting for it (the split layout would run them together too)."""
    stub, log, caches = PagedStub(2, 4), [], [None] * 2
    a = Req(log, "a", _prompt(200, 1), 5, caches)           # ends on slot 0 holding 4 pages
    b = Req(log, "b", _prompt(20, 2), 100, caches)          # takes slot 0: 2 pages are enough
    c = Req(log, "c", _prompt(20, 3), 5, caches)
    _run(stub, caches, [[a], [b, c]])
    assert log.index(("finish", "c")) < log.index(("finish", "b"))   # c ran beside b
    assert len(stub.table[0]) <= 3 and ("release", 0) not in log     # trimmed, not evicted


# ---- the Python and the native server over the same paged stub --------------------------------------------------------------------

class PagedSlotStub:
    """The Python twin of tests/native/api_paged_stub_main.cpp: PagedStub's pages with the token rule of test_api_parallel.SlotStub
    (seeded when sampling, EOS after `eos_after` tokens); `events` records the prefills and the slots whose pages are freed."""
    paged = True

    def __init__(self, slots, pages, regular, eos, eos_after):
        self.pool = PagedStub(slots, pages)
        self.slots, self.slot_len = slots, pages * PAGE
        self.regular, self.eos, self.eos_after = regular, eos, eos_after
        self.seed, self.temp, self.produced = [0] * slots, [0.0] * slots, [0] * slots
        self.events = []

    def slot_reserve(self, slot, rows):
        return self.pool.slot_reserve(slot, rows)

    def slot_trim(self, slot, rows):
        self.pool.slot_trim(slot, rows)

    def slot_release(self, slot):
        if self.pool.table[slot]:
            self.events.append(f"FREE {slot}")
        self.slot_trim(slot, 0)

    def free_pages(self):
        return self.pool.free_pages()

    def slot_pages(self, slot):
        return self.pool.slot_pages(slot)

    def slot_prefill(self, slot, tokens, pos):
        assert pos + len(tokens) <= len(self.pool.table[slot]) * PAGE
        self.events.append(f"POS {slot} {pos} {len(tokens)}")

    def slot_copy(self, src, dst, P):
        assert self.pool.slot_reserve(dst, P)

    def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias, **filters):
        self.seed[slot], self.temp[slot], self.produced[slot] = seed, temperature, 0

    def slots_step(self, tokens, pos, active):
        out = []
        for b in range(self.slots):
            if not active[b]:
                out.append(-1)
                continue
            assert pos[b] < len(self.pool.table[b]) * PAGE
            self.produced[b] += 1
            salt = (self.seed[b] % 997) * 31 if self.temp[b] > 0 else 0
            out.append(self.eos if self.produced[b] > self.eos_after else (tokens[b] * 7 + pos[b] * 13 + 5 + salt) % self.regular)
        return out


def _msgs(i):
    return [{"role": "user", "content": f"client {i} says hello " * (i + 1)}]


def _ask(port, body):
    import http.client
    import json
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=60)
    try:
        c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
        return [(ch["message"]["content"], ch["finish_reason"]) for ch in json.loads(c.getresponse().read())["choices"]]
    finally:
        c.close()


def _paged_sequence(port):
    """Requests one after another on 2 slots over 4 pages: a long completion (3 pages); two sampled choices that take both slots,
    trim the first and are both cut for want of a page; a completion that outgrows its slot's pages by evicting the idle one; and
    its follow-up, which reuses the prefix."""
    out = [_ask(port, dict(messages=_msgs(0), max_tokens=150)),
           _ask(port, dict(messages=_msgs(1), n=2, temperature=0.8, seed=7, max_tokens=230))]
    out.append(_ask(port, dict(messages=_msgs(2), max_tokens=200)))
    out.append(_ask(port, dict(messages=_msgs(2) + [{"role": "assistant", "content": out[-1][0][0]},
                                                  {"role": "user", "content": "more"}], max_tokens=5)))
    return out


def _wait_port(port):
    import socket
    import time
    for _ in range(300):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            return
        except OSError:
            time.sleep(0.02)


def test_python_and_native_servers_agree_on_paged_slots(tmp_path):
    import re
    import socket
    from types import SimpleNamespace
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok_path = str(tmp_path / "t.t")
    write_synthetic_tokenizer(tok_path, 512, style="llama3")
    exe = str(tmp_path / "api_paged_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_paged_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe, "-lpthread"], check=True)

    def free_port():
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        p = s.getsockname()[1]
        s.close()
        return p
    n_req = 4
    port = free_port()
    proc = subprocess.Popen([exe, tok_path, str(port), str(n_req + 1), "2", "4", "1000"], stdout=subprocess.PIPE,
                            stderr=subprocess.STDOUT, text=True)
    _wait_port(port)
    native = _paged_sequence(port)
    try:
        log, _ = proc.communicate(timeout=30)
    except subprocess.TimeoutExpired:
        proc.kill()
        log, _ = proc.communicate()
    assert proc.returncode in (0, None, -9), log
    native_events = re.findall(r"^((?:POS|FREE) [\d ]+)$", log, re.M)

    H = host()
    tok = H.Tokenizer(tok_path)
    model = PagedSlotStub(2, 4, tok.regular_vocab_size, list(tok.eos_ids)[0], 1000)
    port = free_port()
    args = parse_args(["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0",
                       "--parallel", "2", "--parallel-cache", "paged"], False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 77),
                          header=SimpleNamespace(seq_len=256, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, n_req + 1), daemon=True)
    th.start()
    _wait_port(port)
    python = _paged_sequence(port)
    assert python == native
    assert [e.strip() for e in native_events] == model.events
    # what the sequence is meant to show: the sampled choices were cut, the third completion evicted slot 1's cache and ran its
    # 200 tokens, and its follow-up reused its prefix
    assert all(len(t) < len(native[2][0][0]) for t, _ in native[1])
    assert "FREE 1" in native_events
    assert re.search(r"POS 0 [1-9]\d* ", "\n".join(native_events))
