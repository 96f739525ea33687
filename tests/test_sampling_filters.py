"""Sampling filters top_k / min_p: the host Sampler, both API servers, the CLI flags and the tensor-parallel control op.

* The host Sampler against an independent numpy implementation of the rule (README "Chat API: sampling filters"), the same token
  for the same coin over a grid of top_k, min_p, top_p, penalties and bias, with ties at the K-th value.
* Both servers over stub models that draw with the sampler they are handed (tests/native/api_filters_stub_main.cpp and
  FiltersStub below, its Python twin): identical responses and logs, with the request's filters reaching every choice and every
  --parallel slot; malformed values are refused with the server still answering.
"""
import json
import os
import socket
import subprocess
import threading
from types import SimpleNamespace

import numpy as np
import pytest

from test_sampling_controls import MSGS, _free_port, _parts, _post, _wait

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
FIX = 1099511627776.0   # 2^40


def _H():
    from distributed_llama_b200 import host
    return host()


# ---- an independent numpy implementation of the draw ------------------------------------------------------------------------

def _fma32(a, b, c):
    """float32 fused multiply-add, correctly rounded: the float64 sum of the exact product and c, with the double-rounding case
    (a sum exactly halfway between two floats) decided by the exact remainder of that sum."""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b                                  # exact: 24 + 24 significant bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)            # TwoSum: p + c == s + err exactly
    r = s.astype(np.float32)
    up = np.nextafter(r, F32(np.inf))
    dn = np.nextafter(r, F32(-np.inf))
    r64 = r.astype(np.float64)
    mid_up = (s > r64) & (s - r64 == (up.astype(np.float64) - r64) / 2)
    mid_dn = (s < r64) & (r64 - s == (r64 - dn.astype(np.float64)) / 2)
    tie = s == r64
    r = np.where(mid_up & (err > 0), up, r)
    r = np.where(mid_dn & (err < 0), dn, r)
    # s exactly representable but the true value is not: the rounding is already right (|err| < half an f32 ulp)
    return np.where(tie, s.astype(np.float32), r).astype(np.float32)


def exp_neg(x):
    """csrc/common/dl_expf.h expNeg in numpy float32."""
    x = np.asarray(x, dtype=np.float32)
    zero = ~(x > F32(-86.0))
    x = np.where(x > 0, F32(0), x).astype(np.float32)
    x = np.where(zero, F32(0), x).astype(np.float32)
    n = np.rint(x * F32(1.44269504088896341)).astype(np.float32)
    r = _fma32(n, F32(-0.693359375), x)
    r = _fma32(n, F32(2.12194440e-4), r)
    p = np.full_like(x, F32(1.9875691500e-4))
    for c in (1.3981999507e-3, 8.3334519073e-3, 4.1665795894e-2, 1.6666665459e-1, 5.0000001201e-1):
        p = _fma32(p, r, F32(c))
    z = (r * r).astype(np.float32)
    y = _fma32(p, z, r)
    y = (y + F32(1.0)).astype(np.float32)
    bits = y.view(np.uint32).astype(np.int64) + (n.astype(np.int64) << 23)
    out = (bits & 0xFFFFFFFF).astype(np.uint32).view(np.float32)
    return np.where(zero, F32(0), out).astype(np.float32)


class XorShift:
    def __init__(self, seed):
        self.s = seed & 0xFFFFFFFFFFFFFFFF

    def coin(self):
        s = self.s
        s ^= s >> 12
        s ^= (s << 25) & 0xFFFFFFFFFFFFFFFF
        s ^= s >> 27
        self.s = s
        u = ((s * 0x2545F4914F6CDD1D) & 0xFFFFFFFFFFFFFFFF) >> 32
        return F32(u >> 8) / F32(16777216.0)


def _fix(p):
    return (np.asarray(p, dtype=np.float32).astype(np.float64) * FIX).astype(np.uint64)


def candidate_set(e, top_k, min_p):
    """S of the filter rule as a boolean mask over the ids: top_k ranks in the order (e desc, id asc), min_p compares e with
    f32(min_p * max e)."""
    V = len(e)
    keep = np.ones(V, dtype=bool)
    if min_p > 0:
        keep &= e >= F32(F32(min_p) * e.max())
    if 0 < top_k < V:
        order = np.lexsort((np.arange(V), -e.astype(np.float64)))
        rank = np.empty(V, dtype=np.int64)
        rank[order] = np.arange(V)
        keep &= rank < top_k
    return keep


def reference_draw(x, T, topp, top_k, min_p, coin):
    """One temperature > 0 draw from the (controlled) logits x, following the rule step by step."""
    V = len(x)
    y = (np.asarray(x, dtype=np.float32) / F32(T)).astype(np.float32)
    e = exp_neg((y - y.max()).astype(np.float32))
    S = candidate_set(e, top_k, min_p) if (0 < top_k < V or min_p > 0) else np.ones(V, dtype=bool)
    nS = int(S.sum())
    e = np.where(S, e, F32(0)).astype(np.float32)
    total = np.array([int(_fix(e).sum())], dtype=np.uint64).astype(np.float32)[0]
    inv = F32(1.0) / F32(total / F32(FIX))
    p = (e * inv).astype(np.float32)
    if nS == 1:
        return int(np.argmax(S))
    fp = _fix(p)
    if topp <= 0 or topp >= 1:
        cdf = np.cumsum(fp)
        hit = np.nonzero(int(_fix(coin)) < cdf)[0]
        return int(hit[0]) if len(hit) else V - 1
    cutoff = F32(F32(1.0) - F32(topp)) / F32(nS - 1)
    ids = np.nonzero(p >= cutoff)[0]
    ids = ids[np.lexsort((ids, -p[ids].astype(np.float64)))]
    cum = np.cumsum(fp[ids])
    over = np.nonzero(cum > int(_fix(F32(topp))))[0]
    last = int(over[0]) if len(over) else len(ids) - 1
    r = int(_fix(F32(coin * F32(F32(float(cum[last])) / F32(FIX)))))
    hit = np.nonzero(r < cum[:last + 1])[0]
    return int(ids[hit[0]]) if len(hit) else int(ids[last])


def tied_logits(rs, V):
    """Logits with many exact ties (so the K-th value is usually shared) and a few distinct large values."""
    x = (rs.randint(0, 24, V) * 0.5).astype(np.float32)
    x[rs.randint(0, V, 5)] += np.float32(3.0)
    return x


def _controlled(x, counts, bias, presence, frequency):
    x = x.copy()
    if bias:
        b = np.zeros_like(x)
        for t, v in bias:
            b[t] = F32(v)
        x = (x + b).astype(np.float32)
    hit = counts > 0
    x[hit] = ((x[hit] - counts[hit].astype(np.float32) * F32(frequency)) - F32(presence)).astype(np.float32)
    return x


GRID = [(k, 0.0) for k in (1, 2, 40)] + [(0, p) for p in (0.01, 0.5, 1.0)] + [(40, 0.01), (2, 0.5)]


@pytest.mark.parametrize("V", [1000, 32003])
@pytest.mark.parametrize("topp", [0.9, 1.0])
def test_host_sampler_matches_numpy_rule(V, topp):
    H = _H()
    grid = GRID + [(V - 1, 0.0), (V, 0.0), (V + 5, 0.0), (V - 1, 0.01)]
    for g, (top_k, min_p) in enumerate(grid):
        for controls in (False, True):
            seed = 1000 * g + V + (7 if controls else 0)
            T = 0.8 if g % 2 else 1.3
            rs = np.random.RandomState(seed)
            smp = H.Sampler(V, T, topp, seed)
            bias = sorted({int(t): float(F32(v)) for t, v in zip(rs.randint(0, V, 8), rs.uniform(-3, 3, 8))}.items()) if controls else []
            presence, frequency = (0.5, 0.25) if controls else (0.0, 0.0)
            smp.set_controls(presence, frequency, bias)
            smp.set_filters(top_k, min_p)
            ref_rng = XorShift(seed)
            counts = np.zeros(V, dtype=np.int64)
            for d in range(12):
                x = tied_logits(rs, V) if d % 2 else (rs.standard_normal(V) * 3).astype(np.float32)
                want = reference_draw(_controlled(x, counts, bias, presence, frequency) if controls else x, T, topp, top_k, min_p,
                                      ref_rng.coin())
                got = int(smp.sample(x))
                assert got == want, (top_k, min_p, controls, d)
                if controls:
                    counts[got] += 1
                if top_k == 1:   # the arg-max of e, lowest id among ties
                    y = (x if not controls else None)
                    if y is not None:
                        ys = (y / F32(T)).astype(np.float32)
                        e = exp_neg((ys - ys.max()).astype(np.float32))
                        assert got == int(np.argmax(e))


def test_filters_off_draw_exactly_as_before():
    """top_k 0 (or >= V) and min_p 0 leave every draw as it was: the same generator stream and the same tokens."""
    H = _H()
    V = 5000
    rs = np.random.RandomState(3)
    xs = [(rs.standard_normal(V) * 2).astype(np.float32) for _ in range(40)]
    base = H.Sampler(V, 0.9, 0.9, 77)
    ref = [base.sample(x) for x in xs]
    for k, p in ((0, 0.0), (V, 0.0), (V + 1, 0.0), (2**31 - 1, 0.0)):
        s = H.Sampler(V, 0.9, 0.9, 77)
        s.set_filters(k, p)
        assert not s.filters_active
        assert [s.sample(x) for x in xs] == ref


def test_greedy_ignores_filters_and_coin_is_drawn_once():
    H = _H()
    V = 300
    rs = np.random.RandomState(5)
    x = rs.standard_normal(V).astype(np.float32)
    g = H.Sampler(V, 0.0, 0.9, 1)
    g.set_filters(3, 0.5)
    assert g.sample(x) == int(np.argmax(x))
    # top_k = 1 returns the arg-max and advances the generator by one coin, like any draw
    a, b = H.Sampler(V, 0.8, 0.9, 9), H.Sampler(V, 0.8, 0.9, 9)
    a.set_filters(1, 0.0)
    assert a.sample(x) == int(np.argmax(x))
    b.sample(x)
    assert a.next_coin() == b.next_coin()


def test_set_filters_refuses_bad_min_p():
    s = _H().Sampler(10, 0.8, 0.9, 1)
    for bad in (-0.01, 1.01, float("nan")):
        with pytest.raises(ValueError):
            s.set_filters(0, bad)
    s.set_filters(5, 1.0)
    assert (s.top_k, s.min_p) == (5, 1.0)


# ---- both servers ------------------------------------------------------------------------------------------------------------

class FiltersStub:
    """tests/native/api_filters_stub_main.cpp in Python."""
    comm = None

    def __init__(self, V: int, eos: int, slots: int = 0, eos_after: int = 12):
        self.V, self.eos, self.eos_after = V, eos, eos_after
        self.end, self.last, self.log = 0, None, []
        self.slots = slots
        self.slot_len = 4096 // slots if slots else 0
        self.smp = [None] * max(slots, 1)
        self.start = [0] * max(slots, 1)
        self.t_hash = (np.arange(V, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)

    def _logits(self, token, pos, n):
        k = ((self.t_hash[:n] + np.uint64(token * 97 + pos * 13)) & np.uint64(0xFFFFFFFF)) % np.uint64(1000)
        return k.astype(np.float32) / np.float32(100.0)

    def prefill(self, tokens, pos):
        self.log.append(f"POS {pos} {len(tokens)}")
        self.end = pos + len(tokens)

    def next_token(self, token, pos, sampler):
        if sampler.completion_generation != self.last:
            self.last = sampler.completion_generation
            self.log.append(f"FLT {sampler.top_k} {sampler.min_p:.9g}")
        if pos + 1 - self.end > self.eos_after:
            return self.eos
        return int(sampler.sample(self._logits(token, pos, sampler.vocab_size)))

    def forget_device_seed(self):
        pass

    def save_sampler(self):
        return None

    def restore_sampler(self, saved):
        pass

    def batched_choices(self, n):
        return False

    # --parallel
    def slot_prefill(self, slot, tokens, pos):
        self.log.append(f"POS {slot} {pos} {len(tokens)}")
        self.start[slot] = pos + len(tokens)

    def slot_copy(self, src, dst, P):
        self.start[dst] = self.start[src]

    def slot_sampling(self, slot, seed, temperature, topp, presence, frequency, bias, top_k=0, min_p=0.0):
        self.log.append(f"SEED {slot} {seed}")
        s = _H().Sampler(self.V, temperature, topp, seed)
        s.set_controls(presence, frequency, list(bias))
        if top_k or min_p:
            self.log.append(f"SLOTFLT {slot} {top_k} {float(F32(min_p)):.9g}")
            s.set_filters(top_k, min_p)
        self.smp[slot] = s

    def slots_step(self, tokens, pos, active):
        out = [-1] * self.slots
        for s in range(self.slots):
            if not active[s]:
                continue
            if pos[s] + 1 - self.start[s] > self.eos_after:
                out[s] = self.eos
            else:
                out[s] = int(self.smp[s].sample(self._logits(tokens[s], pos[s], self.V)))
        return out


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("api_filters"))
    exe = os.path.join(d, "api_filters_stub")
    srcs = [os.path.join(ROOT, "tests", "native", "api_filters_stub_main.cpp"), os.path.join(ROOT, "csrc", "app", "api_server.cpp"),
            os.path.join(ROOT, "csrc", "host", "text.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wno-sign-compare", *srcs, "-o", exe, "-lpthread"], check=True)
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    tok = os.path.join(d, "t.t")
    write_synthetic_tokenizer(tok, 512, style="llama3")
    return exe, tok


def _flags(top_k, min_p):
    return (["--top-k", str(top_k)] if top_k else []) + (["--min-p", repr(min_p)] if min_p else [])


def _run_python(tok_path, bodies, slots=0, top_k=0, min_p=0.0):
    from distributed_llama_b200.apps import api_server as py_api
    from distributed_llama_b200.apps.args import parse_args
    H = _H()
    tok = H.Tokenizer(tok_path)
    model = FiltersStub(tok.vocab_size, list(tok.eos_ids)[0], slots)
    port = _free_port()
    argv = ["--model", "stub.m", "--tokenizer", tok_path, "--host", "127.0.0.1", "--port", str(port), "--temperature", "0"]
    argv += (["--parallel", str(slots)] if slots else []) + _flags(top_k, min_p)
    args = parse_args(argv, False)
    ctx = SimpleNamespace(args=args, sess=None, inference=model, tokenizer=tok, sampler=H.Sampler(tok.vocab_size, 0.0, 0.9, 0),
                          header=SimpleNamespace(seq_len=4096, vocab_size=tok.vocab_size))
    th = threading.Thread(target=py_api.serve, args=(ctx, len(bodies) + 1), daemon=True)   # + the readiness probe
    th.start()
    _wait(port)
    out = [_post(port, b) for b in bodies]
    th.join(timeout=20)
    return out, model.log


def _run_native(stub, bodies, slots=0, top_k=0, min_p=0.0):
    import re
    exe, tok_path = stub
    port = _free_port()
    cmd = [exe, tok_path, str(port), str(len(bodies) + 1), str(slots or 1)] + _flags(top_k, min_p)
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        _wait(port)
        out = [_post(port, b) for b in bodies]
    finally:
        try:
            log, _ = proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            log, _ = proc.communicate()
    return out, re.findall(r"POS [\d ]+|FLT [^\n]*|SEED \d+ \d+|SLOTFLT [^\n]*", log)


def _cell(**kw):
    return dict(kw, messages=MSGS)


VALID = [
    _cell(temperature=0.8, seed=3, top_k=1),
    _cell(temperature=0.8, seed=3, top_k=2, max_tokens=6),
    _cell(temperature=0.8, seed=3, min_p=0.5),
    _cell(temperature=1.3, seed=4, top_k=40, min_p=0.01, top_p=1.0),
    _cell(temperature=0.8, seed=5, n=3, top_k=3, min_p=0.2, max_tokens=5),
    _cell(temperature=0.8, seed=6, top_k=2147483647, stream=True),
    _cell(temperature=1.0, seed=7, min_p=1, presence_penalty=0.5, logit_bias={"9": 2.5}),
    _cell(temperature=0, top_k=5, min_p=0.3, n=2),
    _cell(temperature=0.9, seed=8, n=2, top_k=0, min_p=0, stream=True, max_tokens=4),
    _cell(temperature=0.7, seed=9, top_k=600, min_p=0.0001),
]


def _check_same(py, nat):
    for i, (a, b) in enumerate(zip(py, nat)):
        assert a, i
        assert _parts(a) == _parts(b), i


def test_servers_agree_on_filtered_completions(stub):
    py, py_log = _run_python(stub[1], VALID)
    nat, nat_log = _run_native(stub, VALID)
    _check_same(py, nat)
    assert py_log == nat_log
    flt = [ln for ln in py_log if ln.startswith("FLT ")]
    assert flt[0] == "FLT 1 0" and flt[2] == "FLT 0 0.5" and flt[3] == "FLT 40 0.00999999978"
    # n = 3: every choice draws with the request's filters
    assert sum(1 for ln in flt if ln == "FLT 3 0.200000003") == 3


def test_top_k_1_is_the_greedy_completion(stub):
    """At temperature > 0, top_k = 1 always draws the arg-max: the stub's greedy completion (its logits have no ties at the top
    that greedy and the filter would order differently)."""
    g, _ = _run_python(stub[1], [_cell(temperature=0, max_tokens=8)])
    k1, _ = _run_python(stub[1], [_cell(temperature=1.5, seed=123, top_k=1, max_tokens=8)])
    assert json.loads(g[0])["choices"][0]["message"] == json.loads(k1[0])["choices"][0]["message"]


def test_servers_agree_under_parallel_slots(stub):
    bodies = [_cell(temperature=0.8, seed=3, n=2, top_k=2, min_p=0.1, max_tokens=5), _cell(temperature=0.8, seed=4, max_tokens=5),
              _cell(temperature=1.1, seed=5, n=3, min_p=0.25, max_tokens=4, stream=True), _cell(temperature=0, top_k=7, max_tokens=3)]
    py, py_log = _run_python(stub[1], bodies, slots=4)
    nat, nat_log = _run_native(stub, bodies, slots=4)
    _check_same(py, nat)
    assert py_log == nat_log
    slot_flt = [ln for ln in py_log if ln.startswith("SLOTFLT ")]
    # every slot of a filtered request gets its filters; an unfiltered request sets none (slot_sampling switched them off)
    assert len([ln for ln in slot_flt if ln.endswith(" 2 0.100000001")]) == 2
    assert len([ln for ln in slot_flt if ln.endswith(" 0 0.25")]) == 3
    assert len([ln for ln in slot_flt if ln.endswith(" 7 0")]) == 1


def test_server_defaults_apply_and_requests_override(stub):
    bodies = [_cell(temperature=0.8, seed=3, max_tokens=4), _cell(temperature=0.8, seed=3, top_k=0, min_p=0, max_tokens=4)]
    py, py_log = _run_python(stub[1], bodies, top_k=3, min_p=0.125)
    nat, nat_log = _run_native(stub, bodies, top_k=3, min_p=0.125)
    _check_same(py, nat)
    assert py_log == nat_log
    assert [ln for ln in py_log if ln.startswith("FLT ")] == ["FLT 3 0.125", "FLT 0 0"]


INVALID = [
    {"top_k": -1}, {"top_k": 2**31}, {"top_k": 1.5}, {"top_k": 40.0}, {"top_k": 4e1}, {"top_k": "40"}, {"top_k": True},
    {"top_k": None}, {"top_k": [1]}, {"min_p": -0.01}, {"min_p": 1.0001}, {"min_p": "0.1"}, {"min_p": False}, {"min_p": None},
    {"min_p": {}}, {"min_p": 1e300},
]


@pytest.mark.parametrize("server", ["python", "native"])
def test_invalid_filters_are_refused(stub, server):
    bad = [_cell(temperature=0.8, **b) for b in INVALID]
    ok = _cell(temperature=0.8, seed=1, max_tokens=3, top_k=5)
    bodies = [x for b in bad for x in (b, ok)]
    out, log = _run_python(stub[1], bodies) if server == "python" else _run_native(stub, bodies)
    for i in range(0, len(bodies), 2):
        assert out[i] == "", bodies[i]
        assert json.loads(out[i + 1])["usage"]["completion_tokens"] == 3, bodies[i]
    assert sum(1 for ln in log if ln.startswith("POS ")) == len(bad)


def test_parse_filters_edges():
    from distributed_llama_b200.apps.api_server import parse_filters
    assert parse_filters({}, 4, 0.5) == (4, 0.5)
    assert parse_filters({"top_k": 0, "min_p": 0}, 4, 0.5) == (0, 0.0)
    assert parse_filters({"top_k": 2**31 - 1, "min_p": 1}, 0, 0.0) == (2**31 - 1, 1.0)


# ---- CLI flags ----------------------------------------------------------------------------------------------------------------

def test_python_cli_flags():
    from distributed_llama_b200.apps.args import USAGE, parse_args
    a = parse_args(["inference", "--top-k", "40", "--min-p", "0.05"], True)
    assert (a.top_k, a.min_p) == (40, 0.05)
    d = parse_args(["inference"], True)
    assert (d.top_k, d.min_p) == (0, 0.0)
    for argv in (["--top-k", "-1"], ["--top-k", "2147483648"], ["--top-k", "1.5"], ["--min-p", "1.5"], ["--min-p", "-0.1"]):
        with pytest.raises(ValueError):
            parse_args(["inference"] + argv, True)
    assert "--top-k" in USAGE and "--min-p" in USAGE
    from distributed_llama_b200.apps import api_server
    assert "--top-k" in api_server.USAGE and "--min-p" in api_server.USAGE


@pytest.mark.parametrize("exe", ["dllama-native", "dllama-api-native"])
def test_native_cli_flags(exe):
    path = os.path.join(ROOT, "distributed_llama_b200", exe)
    if not os.path.exists(path):
        pytest.skip("native binaries are built by build()")
    usage = subprocess.run([path, "--help"], capture_output=True, text=True, timeout=60)
    assert "--top-k" in usage.stdout + usage.stderr and "--min-p" in usage.stdout + usage.stderr
    for bad in (["--top-k", "-3"], ["--top-k", "2147483648"], ["--min-p", "2"]):
        r = subprocess.run([path] + (["inference"] if exe == "dllama-native" else []) + bad, capture_output=True, text=True, timeout=60)
        assert r.returncode != 0
        assert ("--top-k" in r.stdout + r.stderr) or ("--min-p" in r.stdout + r.stderr)


# ---- tensor-parallel control op -----------------------------------------------------------------------------------------------

def test_filters_op_round_trips_over_gloo(tmp_path):
    """RootInference.set_filters sends OP_FILTERS once per change; worker_loop applies the very same (top_k, min_p bits)."""
    import torch.multiprocessing as mp
    port = _free_port()
    q = mp.get_context("spawn").SimpleQueue()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_rank, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
    results = {}
    while not q.empty():
        r, v = q.get()
        results[r] = v
    assert results.get(1) == [(40, 0.05000000074505806), (0, 0.0), (7, 1.0)], results
    assert results.get(0) == results.get(1)


def _gloo_rank(rank, port, q):
    import torch
    import torch.distributed as dist
    from distributed_llama_b200 import host
    from distributed_llama_b200.apps import runtime
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=2)
    seen = []

    class Eng:
        def set_sampling_filters(self, k, p):
            seen.append((int(k), float(np.float32(p))))

    sess = SimpleNamespace(engine=Eng(), header=None, device="cpu")
    if rank == 0:
        inf = runtime.RootInference(sess, SimpleNamespace(rank=0, world_size=2), None)
        smp = host().Sampler(100, 0.8, 0.9, 1)
        for k, p in ((40, 0.05), (40, 0.05), (0, 0.0), (7, 1.0)):
            smp.set_filters(k, p)
            inf.set_filters(smp)   # the repeated setting sends nothing
        inf._send(runtime.OP_STOP, 0, [])
    else:
        runtime.worker_loop(sess, SimpleNamespace(rank=1, world_size=2), None)
    q.put((rank, seen))
    dist.destroy_process_group()
