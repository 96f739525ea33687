"""Per-token log-probabilities on the device (csrc/cuda/logprobs.cu) and their paths up to the chat API.

* Kernel against float64: random rows at V in {257, 32000, 128256, 151936} with 1, 3 and 8 rows per launch; every logprob within
  1e-5 + 1e-6 |ref| of float64 log_softmax, top-k ids equal to the float64 order (value desc, id asc). Ties at the maximum, a
  constant row, spreads of +-1e4, ids >= V excluded, k = 0, 1 and 20, a chosen token outside the top k, and controls (bias,
  counts read after the draw, penalties) against float64 of the transformed row.
* Determinism: a row's block is bitwise the same across launches and beside other rows.
* Engine: the tokens with and without logprobs are equal (greedy on the persistent kernel, sampled on the device sampler), the
  greedy token is top_logprobs[0], the numbers match float64 of the step's own logits and the q80-activation oracle loosely.
* Choices, the MoE fallback and the slots step; the Python chat server end to end.
"""
import http.client
import json
import os
import socket
import subprocess
import sys
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _decode(block):
    from distributed_llama_b200.ops import cuda_lib as cl
    return cl.decode_logprobs(block)


def _ref(x, k):
    """float64 log_softmax of the float32 row x and its k largest entries in the order (value desc, id asc)."""
    x64 = x.astype(np.float64)
    m = x64.max()
    lp = x64 - (m + np.log(np.exp(x64 - m).sum()))
    order = np.lexsort((np.arange(len(x)), -x))[:k]
    return lp, [int(i) for i in order]


def _within(got, want):
    return abs(got - want) <= 1e-5 + 1e-6 * abs(want)


def _check(block, x, k, chosen):
    tok, lp, top = _decode(block)
    ref, order = _ref(x, k)
    assert tok == chosen
    assert _within(lp, ref[chosen]), (lp, ref[chosen])
    assert [i for i, _ in top] == order
    for i, v in top:
        assert _within(v, ref[i]), (i, v, ref[i])
        if i == chosen:
            assert np.float32(v).tobytes() == np.float32(lp).tobytes()


def _controlled(lg, counts, bias, presence, frequency):
    x = lg + bias if bias is not None else lg.copy()
    hit = counts > 0
    x[hit] = (x[hit] - counts[hit].astype(np.float32) * np.float32(frequency)) - np.float32(presence)
    return x


def _run(logits, chosen, ks, **kw):
    from distributed_llama_b200.runtime.engine import logprobs_rows
    out = logprobs_rows(torch.from_numpy(logits).cuda(), torch.tensor(chosen, dtype=torch.int32, device="cuda"), ks, **kw)
    return out.cpu().numpy()


@pytest.mark.parametrize("V", [257, 32000, 128256, 151936])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_kernel_matches_float64(V, B):
    rs = np.random.RandomState(V + B)
    x = (rs.randn(B, V) * 4).astype(np.float32)
    ks = [(0, 1, 5, 20)[b % 4] for b in range(B)]
    chosen = [int(rs.randint(V)) for _ in range(B)]   # mostly outside the top k
    out = _run(x, chosen, ks)
    for b in range(B):
        _check(out[b], x[b], ks[b], chosen[b])


def test_kernel_ties_flat_rows_and_spreads():
    V = 32000
    rs = np.random.RandomState(1)
    rows = []
    r = (rs.randn(V) * 2).astype(np.float32)
    r[rs.choice(V, 300, replace=False)] = 9.5            # many exact ties at the maximum: the lowest ids come first
    rows.append(r)
    rows.append(np.full(V, 0.25, dtype=np.float32))      # constant row
    rows.append((rs.uniform(-1e4, 1e4, V)).astype(np.float32))   # most exp terms underflow
    r = (rs.randn(V) * 3).astype(np.float32)
    r[rs.choice(V, 40, replace=False)] = -0.0            # -0 and +0 are one value
    r[rs.choice(V, 40, replace=False)] = 0.0
    r[:] = np.minimum(r, 0.0)
    rows.append(r)
    x = np.stack(rows)
    chosen = [int(np.argmax(x[0])), 123, int(np.argmax(x[2])), 5]
    for ks in ([20, 20, 20, 20], [1, 1, 1, 1], [0, 0, 0, 0]):
        out = _run(x, chosen, ks)
        for b in range(len(rows)):
            _check(out[b], x[b], ks[b], chosen[b])


def test_kernel_ignores_ids_beyond_the_vocabulary():
    V, W = 1000, 1024
    rs = np.random.RandomState(2)
    x = rs.randn(2, W).astype(np.float32)
    x[:, V] = 50.0                                       # the largest logit sits at V, outside the sampled vocabulary
    from distributed_llama_b200.runtime.engine import logprobs_rows
    dev = torch.from_numpy(x).cuda()
    out = logprobs_rows(dev[:, :V], torch.tensor([3, 4], dtype=torch.int32, device="cuda"), [20, 20]).cpu().numpy()
    for b in range(2):
        _check(out[b], x[b, :V], 20, 3 + b)


@pytest.mark.parametrize("per_row", [False, True])
def test_kernel_with_controls(per_row):
    """Counts are those after the draw: the chosen id's count holds one draw the row did not see (frequency != 0 shows it)."""
    V, B = 32000, 4
    rs = np.random.RandomState(3 + per_row)
    lg = (rs.randn(B, V) * 3).astype(np.float32)
    bias = np.zeros((B, V) if per_row else V, dtype=np.float32)
    idx = rs.choice(V, 100, replace=False)
    if per_row:
        bias[:, idx] = rs.uniform(-100, 100, (B, 100)).astype(np.float32)
    else:
        bias[idx] = rs.uniform(-100, 100, 100).astype(np.float32)
    before = np.zeros((B, V), dtype=np.uint32)
    for b in range(B):
        hit = rs.choice(V, 2000, replace=False)
        before[b, hit] = rs.randint(1, 6, 2000)
    params = np.array([[0.8, 0.9, 0.5 * b - 0.7, 1.5 - 0.6 * b] for b in range(B)], dtype=np.float32)
    presence, frequency = 0.75, 1.25
    chosen = [int(rs.randint(V)) for _ in range(B)]
    chosen[1] = int(np.flatnonzero(before[1])[0])        # a token drawn before too
    after = before.copy()
    for b in range(B):
        after[b, chosen[b]] += 1
    kw = dict(bias=torch.from_numpy(bias).cuda(), counts=torch.from_numpy(after.view(np.int32)).cuda())
    if per_row:
        kw["row_params"] = torch.from_numpy(params).cuda()
    else:
        kw.update(presence=presence, frequency=frequency)
    out = _run(lg, chosen, [20] * B, **kw)
    for b in range(B):
        p, f = (params[b, 2], params[b, 3]) if per_row else (presence, frequency)
        x = _controlled(lg[b], before[b], bias[b] if per_row else bias, p, f)
        _check(out[b], x, 20, chosen[b])


def test_kernel_is_deterministic_and_row_independent():
    V = 128256
    rs = np.random.RandomState(4)
    x = (rs.randn(8, V) * 5).astype(np.float32)
    chosen = [int(rs.randint(V)) for _ in range(8)]
    a = _run(x, chosen, [20] * 8)
    for _ in range(3):
        assert np.array_equal(_run(x, chosen, [20] * 8), a)
    alone = _run(x[5:6], chosen[5:6], [20])
    assert np.array_equal(alone[0], a[5])
    masked = _run(x, chosen, [20] * 8, row_mask=0b00100000)
    assert np.array_equal(masked[5], a[5])
    assert not masked[0].any()                           # rows outside the mask are not written


# ---- engine paths -----------------------------------------------------------------------------------------------------------

def _session(tmp_models, name, T=0.0, seed=4242, kv="bf16", **kw):
    from distributed_llama_b200.api import InferenceSession
    m, t = tmp_models[name]
    return InferenceSession(m, t, temperature=T, topp=0.9, seed=seed, kv_cache_float_type=kv, **kw)


def _decode_loop(s, prompt, steps, k=None):
    toks = s.tokenizer.encode(prompt, True, True)
    s.reset()
    s.prefill(toks[:-1])
    s.sampler.begin_completion()
    tok, out, entries, logits = toks[-1], [], [], []
    for _ in range(steps):
        tok = s.next_token(tok, logprobs=k) if k is not None else s.next_token(tok)
        out.append(tok)
        if k is not None:
            entries.append(s.last_logprobs()[0])
            logits.append(s.engine.logits[0, :s.sampler.vocab_size].float().cpu().numpy())
    return out, entries, logits


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3", "tiny-qwen3-moe"])
@pytest.mark.parametrize("kv", ["bf16", "q80"])
@pytest.mark.parametrize("T", [0.0, 0.8])
def test_engine_single_sequence(tmp_models, name, kv, T):
    s = _session(tmp_models, name, T=T, kv=kv)
    plain, _, _ = _decode_loop(s, "the quick brown fox", 12)
    s.sampler.set_seed(4242)
    s.forget_device_seed()
    got, entries, logits = _decode_loop(s, "the quick brown fox", 12, k=5)
    assert got == plain
    if T == 0.0 and "moe" not in name:
        assert s.engine.mega_active
    for tok, e, x in zip(got, entries, logits):
        assert e[0] == tok
        if T == 0.0:
            assert e[2][0][0] == tok
        ref, order = _ref(x, 5)
        assert _within(e[1], ref[tok])
        assert [i for i, _ in e[2]] == order


def test_engine_against_oracle(tmp_models):
    """The device logprobs of a greedy step are within 0.1 of the q80-activation oracle's log_softmax."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.reference import OracleModel
    name = "tiny-llama31"
    s = _session(tmp_models, name)
    got, entries, _ = _decode_loop(s, "hello there", 6, k=3)
    toks = s.tokenizer.encode("hello there", True, True)
    seq = toks + got[:-1]
    oracle = OracleModel(ModelFile(tmp_models[name][0]), act_quant="q80", device="cuda")
    ref = oracle.forward(seq, 0)[len(toks) - 1:].double()[:, :s.sampler.vocab_size]
    ref = torch.log_softmax(ref, dim=-1).cpu().numpy()
    for j, (tok, e) in enumerate(zip(got, entries)):
        assert abs(e[1] - ref[j][tok]) < 0.1
        for i, v in e[2]:
            assert abs(v - ref[j][i]) < 0.1


def test_choices_rows_match_float64(tmp_models):
    from distributed_llama_b200.api import run_choices
    s = _session(tmp_models, "tiny-llama31", T=0.9)
    toks = s.tokenizer.encode("tell me a story", True, True)
    s.prefill(toks[:-1])
    P = s.pos
    rows = []
    orig_first, orig_step = s.choices_first, s.choices_step

    def grab(fn):
        def f(*a, **kw):
            out = fn(*a, **kw)
            rows.append((out, s.engine.logits[:3, :s.sampler.vocab_size].float().cpu().numpy(), s.last_logprobs()))
            return out
        return f
    s.choices_first, s.choices_step = grab(orig_first), grab(orig_step)
    seen = [[] for _ in range(3)]
    out = run_choices(s, toks[-1], P, 3, 10, s.engine.seq_len, s.sampler, 77, lambda i, t: False, logprobs=4,
                      on_logprobs=lambda i, e: seen[i].append(e))
    s.choices_first, s.choices_step = orig_first, orig_step
    for j, (drawn, lg, entries) in enumerate(rows):
        for b in range(3):
            e = entries[b]
            if e is None:
                continue
            x = lg[0] if j == 0 else lg[b]               # the first draws all read the prompt's row
            ref, order = _ref(x, 4)
            assert e[0] == drawn[b]
            assert _within(e[1], ref[e[0]])
            assert [i for i, _ in e[2]] == order
    for i in range(3):
        assert [e[0] for e in seen[i]] == out[i]
    # the same tokens without logprobs
    s2 = _session(tmp_models, "tiny-llama31", T=0.9)
    s2.prefill(toks[:-1])
    assert run_choices(s2, toks[-1], P, 3, 10, s2.engine.seq_len, s2.sampler, 77, lambda i, t: False) == out


def test_moe_choices_fallback_equals_single_runs(tmp_models):
    from distributed_llama_b200 import host
    from distributed_llama_b200.api import run_choices
    s = _session(tmp_models, "tiny-qwen3-moe", T=0.9)
    toks = s.tokenizer.encode("tell me a story", True, True)
    s.prefill(toks[:-1])
    P = s.pos
    seen = [[] for _ in range(2)]
    run_choices(s, toks[-1], P, 2, 6, s.engine.seq_len, s.sampler, 99, lambda i, t: False, logprobs=3,
                on_logprobs=lambda i, e: seen[i].append(e))
    for i in range(2):
        one = _session(tmp_models, "tiny-qwen3-moe", T=0.9, seed=host().choice_seed(99, i))
        got, entries, _ = _decode_loop(one, "tell me a story", 6, k=3)
        assert [e[0] for e in seen[i]] == got
        assert seen[i] == entries


def test_slots_entries_are_batch_invariant(tmp_models):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    eng = Engine(load_device_weights(ModelFile(tmp_models["tiny-llama31"][0])))
    eng.set_slots(4)
    prompts = [[(11 * b + 7 * i + 3) % 500 + 1 for i in range(4 + 5 * b)] for b in range(4)]
    settings = [(0.0, 0.9, 0.0, 0.0), (0.8, 0.9, 0.5, 1.0), (1.1, 0.0, 0.0, 0.0), (0.7, 0.95, 0.25, -0.5)]

    def run(rows, lp_rows):
        for b in rows:
            eng.slot_prefill(b, prompts[b][:-1], 0)
            eng.slot_sampling(b, 1000 + b, *settings[b], [(b + 3, 2.0)] if b % 2 else [])
            if b in lp_rows:
                eng.slot_logprobs(b, 20)
        tokens = [prompts[b][-1] if b in rows else 0 for b in range(4)]
        pos = [len(prompts[b]) - 1 if b in rows else 0 for b in range(4)]
        active = [b in rows for b in range(4)]
        drawn, ents = {b: [] for b in rows}, {b: [] for b in rows}
        for _ in range(10):
            out, lps = eng.slots_step_logprobs(tokens, pos, active)
            for b in rows:
                drawn[b].append(out[b])
                ents[b].append(lps[b])
                assert (lps[b] is None) == (b not in lp_rows)
                tokens[b], pos[b] = out[b], pos[b] + 1
        return drawn, ents

    all_tok, all_lp = run([0, 1, 2, 3], [0, 1, 3])
    for b in (1, 3):
        tok, lp = run([b], [b])
        assert tok[b] == all_tok[b]
        assert lp[b] == all_lp[b]                      # the same float32 values, bit for bit
    plain, _ = run([0, 1, 2, 3], [])
    assert plain == all_tok


# ---- chat API end to end -------------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _post(port, body):
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
    try:
        c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
        return c.getresponse().read().decode()
    finally:
        c.close()


def _stream_choices(text, n):
    content, entries = [""] * n, [[] for _ in range(n)]
    for line in text.split("\r\n"):
        if not line.startswith("data: {"):
            continue
        c = json.loads(line[6:])["choices"][0]
        if "delta" in c:
            content[c["index"]] += c["delta"]["content"]
            entries[c["index"]] += c["logprobs"]["content"]
    return content, entries


def _has_key(obj, key):
    if isinstance(obj, dict):
        return key in obj or any(_has_key(v, key) for v in obj.values())
    if isinstance(obj, list):
        return any(_has_key(v, key) for v in obj)
    return False


@pytest.mark.parametrize("parallel", [1, 4])
def test_python_server_end_to_end(tmp_models, parallel):
    m, t = tmp_models["tiny-llama31"]
    port = _free_port()
    proc = subprocess.Popen([sys.executable, "-m", "distributed_llama_b200.apps.api_server", "--model", m, "--tokenizer", t, "--port",
                             str(port), "--host", "127.0.0.1", "--parallel", str(parallel)], cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT),
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.5).close()
                break
            except OSError:
                assert proc.poll() is None, proc.stdout.read()
                time.sleep(0.2)
        for n in (1, 3):
            for extra in ({}, {"presence_penalty": 0.5, "frequency_penalty": 1.0, "logit_bias": {"7": 3.0}}):
                base = {"messages": [{"role": "user", "content": "write something long"}], "max_tokens": 16, "temperature": 0.8,
                        "seed": 31, "n": n, **extra}
                plain = json.loads(_post(port, base))
                assert not _has_key(plain, "logprobs")
                full = json.loads(_post(port, dict(base, logprobs=True, top_logprobs=3)))
                streamed = _stream_choices(_post(port, dict(base, logprobs=True, top_logprobs=3, stream=True)), n)
                for i in range(n):
                    ch = full["choices"][i]
                    assert ch["message"]["content"] == plain["choices"][i]["message"]["content"]
                    content = ch["logprobs"]["content"]
                    assert 1 <= len(content) <= 16
                    for e in content:
                        assert set(e) == {"token", "logprob", "bytes", "top_logprobs"}
                        assert len(e["top_logprobs"]) == 3
                        assert bytes(e["bytes"]).decode("utf-8", errors="replace") == e["token"]
                        assert all(a["logprob"] >= b["logprob"] for a, b in zip(e["top_logprobs"], e["top_logprobs"][1:]))
                    assert streamed[0][i] == ch["message"]["content"]
                    assert streamed[1][i] == content
        # malformed fields close the connection; the server keeps serving
        for bad in ({"logprobs": 1}, {"logprobs": True, "top_logprobs": 21}, {"top_logprobs": 2}, {"logprobs": True, "top_logprobs": 1.0}):
            with pytest.raises((http.client.RemoteDisconnected, ConnectionError)):
                _post(port, {"messages": [{"role": "user", "content": "hi"}], "max_tokens": 2, **bad})
        ok = json.loads(_post(port, {"messages": [{"role": "user", "content": "hi"}], "max_tokens": 2, "logprobs": True}))
        assert all(e["top_logprobs"] == [] for e in ok["choices"][0]["logprobs"]["content"])
    finally:
        proc.kill()
        proc.communicate()
