"""Sampling filters top_k / min_p on the device (csrc/cuda/sampler.cu, the engine, choices, slots, servers) against the host Sampler.

* sampleKernel with per-row filters, temperatures, top-p and (half the cases) penalties with random counts, against the host
  Sampler (whose rule tests/test_sampling_filters.py pins to an independent numpy implementation): at least 250 draws per
  setting at V = 32003 and 151936, every draw the same token up to the exp tolerance of test_gpu_sampler.py (one in 250).
  The scalar launch path (launchSample) draws what the per-row path draws.
* Batch invariance: a row's draws are the same alone or beside 7 other rows with other filters.
* Tiny models at T = 0.8: top_k = 1 reproduces the greedy completion on the single-sequence, n-choices and --parallel slot paths;
  at T = 0 the filters leave the persistent kernel and the tokens as they were. Engine draws with filters equal a host loop.
* The native CLI and API server end to end, and tensor parallelism (two GPUs): the same tokens as one GPU.
"""
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROMPT = [3, 17, 250, 9, 44]


def _host():
    from distributed_llama_b200 import host
    return host()


def _row_settings(V, grid):
    # (top_k, min_p, temperature, top-p) of the 8 rows
    Ts = (0.8, 1.3, 0.8, 1.3, 1.0, 0.7, 1.3, 0.9)
    return [(k, p, Ts[b], grid_topp) for b, ((k, p), grid_topp) in enumerate(grid)]


def _grids(V):
    a = [((1, 0.0), 0.9), ((2, 0.0), 0.9), ((40, 0.0), 1.0), ((V - 1, 0.0), 0.9), ((0, 0.01), 0.9), ((0, 0.5), 1.0), ((0, 1.0), 0.9),
         ((40, 0.01), 0.9)]
    b = [((V, 0.0), 0.9), ((V + 5, 0.0), 1.0), ((2, 0.5), 0.9), ((40, 0.0), 0.9), ((0, 0.01), 1.0), ((1, 0.0), 1.0), ((0, 0.5), 0.9),
         ((V - 1, 0.01), 1.0)]
    return {"a": a, "b": b}


def _tied(rs, V):
    x = (rs.randint(0, 24, V) * 0.5).astype(np.float32)
    x[rs.randint(0, V, 5)] += np.float32(3.0)
    return x


def _controlled(lg, counts, presence, frequency):
    x = lg.copy()
    hit = counts > 0
    x[hit] = (x[hit] - counts[hit].astype(np.float32) * np.float32(frequency)) - np.float32(presence)
    return x


def _launch(lib, cl, lg_d, V, n, probs, params_d, filt_d, rng, tok, B, mask, cnt_d):
    assert lib.dl_sample_rows_filtered(lg_d.data_ptr(), V, probs.data_ptr(), n, params_d.data_ptr(), filt_d.data_ptr(), rng.data_ptr(),
                                       tok.data_ptr(), B, mask, None, 0, cnt_d.data_ptr() if cnt_d is not None else None, V,
                                       cl.stream_ptr()) == 0


def _filters_tensor(settings):
    raw = np.zeros(len(settings), dtype=[("k", np.uint32), ("p", np.float32)])
    raw["k"] = [s[0] for s in settings]
    raw["p"] = [s[1] for s in settings]
    return torch.from_numpy(raw.view(np.int32).reshape(-1).copy()).cuda()


@pytest.mark.parametrize("V", [32003, 151936])
@pytest.mark.parametrize("grid", ["a", "b"])
@pytest.mark.parametrize("controls", [False, True])
def test_kernel_matches_host_sampler(V, grid, controls):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib, H = cl.lib(), _host()
    rs = np.random.RandomState(V + (grid == "b") * 7 + controls * 13)
    B, launches = 8, 252
    settings = _row_settings(V, _grids(V)[grid])
    presence, frequency = (0.5, 0.75) if controls else (0.0, 0.0)
    params = torch.tensor([[T, topp, presence, frequency] for (_, _, T, topp) in settings], dtype=torch.float32, device="cuda")
    filt = _filters_tensor(settings)
    counts = np.zeros((B, V), dtype=np.uint32)
    if controls:
        for b in range(B):
            hit = rs.choice(V, 500, replace=False)
            counts[b, hit] = rs.randint(1, 4, 500)
    cnt_d = torch.from_numpy(counts.view(np.int32)).cuda() if controls else None
    seeds = [int(s) for s in rs.randint(1, 2 ** 62, B)]
    rng = torch.tensor(seeds, dtype=torch.int64, device="cuda")
    hs = []
    for (k, p, T, topp), s in zip(settings, seeds):
        h = H.Sampler(V, T, topp, s)
        h.set_filters(k, p)
        hs.append(h)
    probs = torch.empty(B * V + 16, device="cuda")
    tok = torch.zeros(B, dtype=torch.int32, device="cuda")
    agree = np.zeros(B, dtype=np.int64)
    total = np.zeros(B, dtype=np.int64)
    for j in range(launches):
        lg = np.stack([_tied(rs, V) if (j + b) % 2 else (rs.randn(V) * 3).astype(np.float32) for b in range(B)])
        _launch(lib, cl, torch.from_numpy(lg).cuda(), V, V, probs, params, filt, rng, tok, B, 0, cnt_d)
        got = tok.tolist()
        for b in range(B):
            x = _controlled(lg[b], counts[b], presence, frequency) if controls else lg[b]
            want = int(hs[b].sample(x))
            total[b] += 1
            agree[b] += want == got[b]
            if controls:
                counts[b, got[b]] += 1
            if settings[b][0] == 1 and want == got[b]:   # top_k = 1: the arg-max, lowest id among ties
                y = (x / np.float32(settings[b][2])).astype(np.float32)
                assert got[b] == int(np.flatnonzero(y == y.max())[0])
    assert (total >= 250).all()
    assert (agree >= total - 1).all(), (agree, total)


def test_scalar_launch_equals_row_launch():
    """launchSample (the single-sequence path) with filters draws what one row of launchSampleRows draws."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    V = 128256
    rs = np.random.RandomState(1)
    for k, p, T, topp in [(40, 0.05, 0.8, 0.9), (1, 0.0, 1.0, 1.0), (0, 0.1, 1.3, 0.9), (7, 0.0, 0.6, 1.0)]:
        rng_a = torch.tensor([99], dtype=torch.int64, device="cuda")
        rng_b = rng_a.clone()
        probs = torch.empty(V + 16, device="cuda")
        ta, tb = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
        params = torch.tensor([[T, topp, 0.0, 0.0]], dtype=torch.float32, device="cuda")
        filt = _filters_tensor([(k, p)])
        for _ in range(30):
            lg = torch.from_numpy((rs.randn(V) * 3).astype(np.float32)).cuda()
            assert lib.dl_sample_logits_filtered(lg.data_ptr(), probs.data_ptr(), V, T, topp, k, p, rng_a.data_ptr(), ta.data_ptr(),
                                                 cl.stream_ptr()) == 0
            _launch(lib, cl, lg, V, V, probs, params, filt, rng_b, tb, 1, 0, None)
            assert int(ta) == int(tb)
        assert int(rng_a) == int(rng_b)
    # min_p outside [0, 1] is refused
    assert lib.dl_sample_logits_filtered(lg.data_ptr(), probs.data_ptr(), V, 0.8, 0.9, 0, 1.5, rng_a.data_ptr(), ta.data_ptr(),
                                         cl.stream_ptr()) != 0


def test_rows_batch_invariance():
    """A row's draws are the same launched alone (B = 1) or as one of 8 rows with other filters and settings."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    V, B = 151936, 8
    rs = np.random.RandomState(2)
    settings = _row_settings(V, _grids(V)["a"])
    params = torch.tensor([[T, topp, 0.0, 0.0] for (_, _, T, topp) in settings], dtype=torch.float32, device="cuda")
    filt = _filters_tensor(settings)
    seeds = [int(s) for s in rs.randint(1, 2 ** 62, B)]
    lgs = [torch.from_numpy(np.stack([_tied(rs, V) if (j + b) % 2 else (rs.randn(V) * 3).astype(np.float32) for b in range(B)])).cuda()
           for j in range(20)]
    probs = torch.empty(B * V + 16, device="cuda")
    rng = torch.tensor(seeds, dtype=torch.int64, device="cuda")
    tok = torch.zeros(B, dtype=torch.int32, device="cuda")
    together = []
    for lg in lgs:
        _launch(lib, cl, lg, V, V, probs, params, filt, rng, tok, B, 0, None)
        together.append(tok.tolist())
    for b in range(B):
        r1 = torch.tensor([seeds[b]], dtype=torch.int64, device="cuda")
        t1 = torch.zeros(1, dtype=torch.int32, device="cuda")
        p1, f1 = params[b:b + 1].contiguous(), _filters_tensor([settings[b]])
        for j, lg in enumerate(lgs):
            _launch(lib, cl, lg[b].contiguous(), V, V, probs, p1, f1, r1, t1, 1, 0, None)
            assert int(t1) == together[j][b], (b, j)


# ---- the engine -------------------------------------------------------------------------------------------------------------

def _session(tmp_models, name, T, seed=4242, **kw):
    from distributed_llama_b200.api import InferenceSession
    m, t = tmp_models[name]
    return InferenceSession(m, t, temperature=T, topp=0.9, seed=seed, **kw)


def _greedy(tmp_models, name, steps):
    ref = _session(tmp_models, name, 0.0)
    ref.prefill(PROMPT[:-1])
    return ref.engine.decode_greedy(PROMPT[-1], len(PROMPT) - 1, steps)


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_top_k_1_is_greedy_on_every_path(tmp_models, name):
    from distributed_llama_b200.api import run_choices
    steps = 16
    want = _greedy(tmp_models, name, steps)
    # single sequence, T = 0.8
    s = _session(tmp_models, name, 0.8, top_k=1)
    s.prefill(PROMPT[:-1])
    tok, got = PROMPT[-1], []
    for _ in range(steps):
        tok = s.next_token(tok)
        got.append(tok)
    assert got == want
    # n = 3 choices (batched on dense models)
    c = _session(tmp_models, name, 0.8, top_k=1)
    c.prefill(PROMPT[:-1])
    out = run_choices(c, PROMPT[-1], c.pos, 3, steps, c.engine.seq_len, c.sampler, 5, lambda i, t: False)
    assert all(o == want for o in out)
    # min_p = 1 keeps the maximum alone as well (the tiny models have no ties at the top)
    s = _session(tmp_models, name, 1.2, min_p=1.0)
    s.prefill(PROMPT[:-1])
    tok, got = PROMPT[-1], []
    for _ in range(steps):
        tok = s.next_token(tok)
        got.append(tok)
    assert got == want


def test_top_k_1_is_greedy_in_slots(tmp_models):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    steps = 12
    want = _greedy(tmp_models, "tiny-llama31", steps)
    eng = Engine(load_device_weights(ModelFile(tmp_models["tiny-llama31"][0])))
    eng.set_slots(4)
    for b in range(4):
        eng.slot_prefill(b, PROMPT[:-1], 0)
        eng.slot_sampling(b, 100 + b, 0.8, 0.9, top_k=1 if b != 2 else 0, min_p=0.0 if b != 3 else 0.3)
    tokens, pos = [PROMPT[-1]] * 4, [len(PROMPT) - 1] * 4
    drawn = [[] for _ in range(4)]
    for _ in range(steps):
        out = eng.slots_step(tokens, pos, [True] * 4)
        for b in range(4):
            drawn[b].append(out[b])
        tokens, pos = out, [p + 1 for p in pos]
    assert drawn[0] == want and drawn[1] == want and drawn[3] == want
    # a new sequence in a slot starts without filters: slot 0 re-admitted at T = 0.8 without them draws what slot 2 drew
    eng.slot_sampling(0, 102, 0.8, 0.9)
    eng.slot_prefill(0, PROMPT[:-1], 0)
    tokens, pos, again = [PROMPT[-1]] + [0] * 3, [len(PROMPT) - 1] + [0] * 3, []
    for _ in range(steps):
        out = eng.slots_step(tokens, pos, [True, False, False, False])
        again.append(out[0])
        tokens[0], pos[0] = out[0], pos[0] + 1
    assert again == drawn[2]


def test_greedy_with_filters_keeps_the_persistent_kernel(tmp_models):
    steps = 12
    s = _session(tmp_models, "tiny-llama31", 0.0, top_k=5, min_p=0.3)
    s.prefill(PROMPT[:-1])
    tok, got = PROMPT[-1], []
    for _ in range(steps):
        tok = s.next_token(tok)
        got.append(tok)
        assert s.engine.mega_active
    assert s.engine.graph_captured and s._dev_filters == (0, 0.0)   # greedy never hands the filters to the device
    assert got == _greedy(tmp_models, "tiny-llama31", steps)


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3-moe"])
def test_engine_filters_match_host_loop(tmp_models, name):
    H = _host()
    steps = 24
    kw = dict(top_k=40, min_p=0.05)
    dev = _session(tmp_models, name, 0.9, **kw)
    dev.prefill(PROMPT[:-1])
    tok, got = PROMPT[-1], []
    for _ in range(steps):
        tok = dev.next_token(tok)
        got.append(tok)
    ref = _session(tmp_models, name, 0.9)
    ref.prefill(PROMPT[:-1])
    smp = H.Sampler(ref.sampler.vocab_size, 0.9, 0.9, 4242)
    smp.set_filters(40, 0.05)
    tok, want = PROMPT[-1], []
    for _ in range(steps):
        tok = int(smp.sample(ref.forward_logits(tok).float().cpu().numpy()[:smp.vocab_size].copy()))
        want.append(tok)
    assert got == want


# ---- the binaries -----------------------------------------------------------------------------------------------------------

def _pred(exe, m, t, extra, gpus=1):
    argv = [os.path.join(ROOT, exe), "inference", "--model", m, "--tokenizer", t, "--prompt", "Hello world", "--steps", "32"] + extra
    r = subprocess.run(argv + (["--gpus", str(gpus)] if gpus > 1 else []), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    return [ln.split("|")[-1] for ln in r.stdout.splitlines() if "🔶 Pred" in ln]


def test_clis_top_k_1_equal_greedy(tmp_models):
    m, t = tmp_models["tiny-llama31"]
    greedy = _pred("dllama-native", m, t, ["--temperature", "0"])
    assert len(greedy) >= 8
    assert _pred("dllama-native", m, t, ["--temperature", "0.8", "--seed", "3", "--top-k", "1"]) == greedy
    assert _pred("dllama", m, t, ["--temperature", "0.8", "--seed", "3", "--top-k", "1", "--buffer-float-type", "q80"]) == greedy
    # filtered sampling: the native CLI (host Sampler) and the Python CLI (device sampler) draw the same tokens
    f = ["--temperature", "0.9", "--seed", "11", "--top-k", "20", "--min-p", "0.05"]
    assert _pred("dllama-native", m, t, f) == _pred("dllama", m, t, f + ["--buffer-float-type", "q80"])


def _serve(exe_argv, bodies):
    import http.client
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    proc = subprocess.Popen(exe_argv + ["--host", "127.0.0.1", "--port", str(port)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                            text=True, cwd=ROOT)
    try:
        for _ in range(1200):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
                break
            except OSError:
                time.sleep(0.1)
        out = []
        for body in bodies:
            c = http.client.HTTPConnection("127.0.0.1", port, timeout=300)
            c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
            r = c.getresponse()
            assert r.status == 200
            out.append([ch["message"]["content"] for ch in json.loads(r.read().decode("utf-8"))["choices"]])
        return out
    finally:
        proc.terminate()
        try:
            proc.communicate(timeout=30)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.communicate()


@pytest.mark.parametrize("server", ["dllama-api-native", "dllama-api"])
@pytest.mark.parametrize("parallel", [1, 4])
def test_servers_end_to_end(tmp_models, server, parallel):
    """top_k = 1 at T = 0.8 answers every choice with the greedy completion, on the choices path and under --parallel."""
    m, t = tmp_models["tiny-llama31"]
    base = {"messages": [{"role": "user", "content": "Hello there"}], "max_tokens": 24}
    bodies = [dict(base, temperature=0), dict(base, temperature=0.8, seed=5, n=3, top_k=1),
              dict(base, temperature=1.2, seed=6, n=2, min_p=1.0)]
    argv = [os.path.join(ROOT, server), "--model", m, "--tokenizer", t, "--temperature", "0"]
    argv += ["--max-requests", str(len(bodies) + 1)] if server.endswith("native") else []
    argv += ["--parallel", str(parallel)] if parallel > 1 else []
    greedy, k1, p1 = _serve(argv, bodies)
    assert all(x == greedy[0] for x in k1) and all(x == greedy[0] for x in p1)


# ---- tensor parallelism ----------------------------------------------------------------------------------------------------

@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_filters_tensor_parallel(tmp_models, tmp_path):
    """Sampled tokens with filters under TP = 2 (the device sampler on gathered logits, OP_FILTERS / TP_OP_FILTERS) equal TP = 1."""
    from distributed_llama_b200.api import run_choices
    m, t = tmp_models["tiny-llama31"]
    code = f"""
import json
from distributed_llama_b200.apps.runtime import init_distributed_from_env, open_control_channel, RootInference, worker_loop
from distributed_llama_b200.api import InferenceSession, run_choices
comm = init_distributed_from_env()
sess = InferenceSession({m!r}, {t!r}, temperature=0.9, topp=0.9, seed=7, comm=comm, top_k=20, min_p=0.05)
chan = open_control_channel(comm)
if comm.rank != 0:
    worker_loop(sess, comm, chan)
else:
    inf = RootInference(sess, comm, chan)
    inf.prefill({PROMPT[:-1]!r}, 0)
    out = run_choices(inf, {PROMPT[-1]}, 4, 1, 16, sess.engine.seq_len, sess.sampler, 7, lambda i, t: False)
    inf.finish()
    print("TOKENS " + json.dumps(out[0]))
"""
    script = tmp_path / "tp_filters.py"
    script.write_text(code)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node=2", str(script)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    tp = json.loads(r.stdout.split("TOKENS ")[1].splitlines()[0])
    one = _session(tmp_models, "tiny-llama31", 0.9, seed=7, top_k=20, min_p=0.05)
    one.prefill(PROMPT[:-1])
    assert tp == run_choices(one, PROMPT[-1], 4, 1, 16, one.engine.seq_len, one.sampler, 7, lambda i, t: False)[0]
    f = ["--temperature", "0.9", "--seed", "11", "--top-k", "20", "--min-p", "0.05"]
    assert _pred("dllama-native", m, t, f, gpus=2) == _pred("dllama-native", m, t, f)
