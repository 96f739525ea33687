"""Independent sequences in KV-cache slots (csrc/cuda/attn_decode.cu, the engine's slots step, per-row sampling).

* slotAttnKernel against a float64 reference over the same bf16 cache, rows at different positions in different slots. "Needle"
  keys parallel to a row's first q-head sit on both sides of its split boundaries, and in the neighbouring slots at rows the
  row would see if it read outside its slot: a lost split, or a read outside the slot, moves the output far beyond the bound.
  Tolerance 2e-4 * max|V|, the bound of tests/test_gpu_choices.py.
* The engine's slots step, teacher-forced, against OracleModel at the tolerance of test_engine_matches_oracle.
* Batch invariance: a row's logits are bitwise those of the same sequence stepped with every other slot idle.
* Per-row sampling settings against the host Sampler with the same seeds.
* dllama-api --parallel 4 end to end: concurrent greedy requests return what each returns alone.
"""
import http.client
import json
import math
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
TOL_V = 2e-4
NEEDLE_SCORE = 30.0
N_SPLITS = 8


def _split_bounds(p: int):
    n_pos = p + 1
    eff = max(1, min(N_SPLITS, (n_pos + 63) // 64))
    chunk = (n_pos + eff - 1) // eff
    return [s * chunk for s in range(1, eff) if s * chunk < n_pos]


@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4), (64, 4), (128, 1)])
@pytest.mark.parametrize("B", [1, 2, 3, 5, 8])
def test_slot_attention_matches_float64(B, hd, kv_mul):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    L = 1024
    g = torch.Generator().manual_seed(B * 17 + hd + kv_mul * 3)
    n_kv = 2
    n_heads = n_kv * kv_mul
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    qkv_dim = q_dim + 2 * kv_dim
    choices = [0, 63, 64, 300, L - 1, 511, 127, 700]
    pos = [choices[(b * 3 + hd // 64) % len(choices)] for b in range(B)]
    inactive = 0b10 if B >= 3 else 0                       # row 1 idle: it must not disturb the others
    qkv = torch.randn(B, qkv_dim, generator=g)
    k = (torch.randn(B, n_kv, L, hd, generator=g) * 0.6).to(torch.bfloat16)
    v = torch.randn(B, n_kv, L, hd, generator=g).to(torch.bfloat16)
    scale = 1.0 / math.sqrt(hd)
    for b in range(B):
        q0 = qkv[b, :hd].double()                          # q-head 0 of KV head 0
        needle = (q0 * (NEEDLE_SCORE / (scale * float(q0 @ q0)))).to(torch.bfloat16)
        for r in [0, pos[b]] + _split_bounds(pos[b]) + [x - 1 for x in _split_bounds(pos[b])]:
            k[b, 0, r] = needle * 0.5                      # inside the slot: must be weighted correctly
        for nb_ in (b - 1, b + 1):                         # outside the slot: must not be read at all
            if 0 <= nb_ < B:
                for r in {0, pos[b] // 2, pos[b]}:
                    k[nb_, 0, r] = needle
    kd, vd = k.cuda().contiguous(), v.cuda().contiguous()
    qd = qkv.cuda().contiguous()
    posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
    partial = torch.zeros(B * n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(B * n_kv, dtype=torch.int32, device="cuda")
    out = torch.full((B, q_dim), float("nan"), device="cuda")
    assert lib.dl_slot_attn(qd.data_ptr(), qkv_dim, posd.data_ptr(), kd.data_ptr(), vd.data_ptr(), n_heads, n_kv, hd, L, N_SPLITS, B,
                            inactive, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    got = out.cpu().double()
    assert int(counters.abs().sum()) == 0                  # self-resetting
    for b in range(B):
        if (inactive >> b) & 1:
            continue
        n = pos[b] + 1
        for h in range(n_heads):
            kvh = h // kv_mul
            q = qkv[b, h * hd:(h + 1) * hd].double()
            s = (k[b, kvh, :n].double() @ q) * scale
            p = torch.softmax(s, dim=0)
            want = p @ v[b, kvh, :n].double()
            err = (got[b, h * hd:(h + 1) * hd] - want).abs().max().item()
            bound = TOL_V * v[b, kvh, :n].double().abs().max().item()
            assert err <= bound, (b, h, pos[b], err, bound)


def _setup(tmp_models, name, slots):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    mf = ModelFile(tmp_models[name][0])
    eng = Engine(load_device_weights(mf))
    eng.set_slots(slots)
    return mf, eng


def _prompts(n, vocab=500):
    return [[(11 * b + 7 * i + 3) % vocab + 1 for i in range(4 + 5 * b)] for b in range(n)]


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_slots_step_matches_oracle(tmp_models, name):
    """Teacher-forced rows against OracleModel at test_engine_matches_oracle's tolerance. At a position where the single-sequence
    engine itself (same prefill kernels, then one token per step) is further from the q80 oracle than that, the row may be as far
    as the single-sequence engine plus a margin: the prefill's bf16 activations and q80 rounding flips, not the slot, set the error."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    from distributed_llama_b200.runtime import Engine
    N = 4
    mf, eng = _setup(tmp_models, name, N)
    prompts = _prompts(N)
    follow = [[(5 * b + 13 * j) % 400 + 2 for j in range(6)] for b in range(N)]
    ref, single = [], []
    for b in range(N):
        seq = prompts[b] + follow[b]
        P = len(prompts[b]) - 1
        ref.append(OracleModel(mf, act_quant="q80", device="cuda").forward(seq, 0)[P:])
        one = Engine(load_device_weights(ModelFile(tmp_models[name][0])))
        one.tc_min_tokens = 1                               # the slot prefill's kernels
        one.prefill(seq[:P], 0, want_logits=False)
        single.append([one.step(seq[p], p).clone() for p in range(P, len(seq))])
        eng.slot_prefill(b, prompts[b][:-1], 0)
    tokens = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    for j in range(len(follow[0]) + 1):
        active = [True] * N
        if j == 3:
            active[2] = False                               # an idle row keeps its slot and position
        lg = eng.slots_forward(tokens, pos, active).clone()
        for b in range(N):
            if not active[b]:
                continue
            step = pos[b] - (len(prompts[b]) - 1)
            err = (lg[b] - ref[b][step]).abs().max().item()
            base = (single[b][step] - ref[b][step]).abs().max().item()
            assert err < max(0.06, base + 0.03), (b, j, err, base)
            # the same prefill kernels, then ordinary single-sequence decode steps: only the attention kernel differs
            assert (lg[b] - single[b][step]).abs().max().item() < 1e-2, (b, j)
            if step < len(follow[b]):
                tokens[b] = follow[b][step]
                pos[b] += 1


def test_slots_batch_invariance(tmp_models):
    """Each row's logits and draws are bit for bit those of the same sequence stepped with every other slot idle."""
    N = 8
    mf, eng = _setup(tmp_models, "tiny-llama31", N)
    prompts = _prompts(N)
    steps = 12
    settings = [(0.0, 0.9), (0.8, 0.9), (1.1, 0.0), (0.0, 0.5), (0.7, 0.95), (0.8, 0.9), (1.3, 0.7), (0.9, 0.9)]

    def run(rows):
        logits, drawn = {b: [] for b in rows}, {b: [] for b in rows}
        for b in rows:
            eng.slot_prefill(b, prompts[b][:-1], 0)
            T, topp = settings[b]
            eng.slot_sampling(b, 1000 + b, T, topp, 0.25 * (b % 3), 0.5 * (b % 2), [(b + 3, 2.0)] if b % 2 else [])
        tokens = [prompts[b][-1] if b in rows else 0 for b in range(N)]
        pos = [len(prompts[b]) - 1 if b in rows else 0 for b in range(N)]
        active = [b in rows for b in range(N)]
        for _ in range(steps):
            lg = eng.slots_forward(tokens, pos, active).clone()
            out = eng.slots_step(tokens, pos, active)       # the same forward again, then the draws
            assert all(torch.equal(eng.logits[b], lg[b]) for b in rows)
            for b in rows:
                logits[b].append(lg[b].cpu())
                drawn[b].append(out[b])
                tokens[b], pos[b] = out[b], pos[b] + 1
        return logits, drawn

    all_lg, all_tok = run(list(range(N)))
    for b in (0, 3, 5, 7):
        lg, tok = run([b])
        assert tok[b] == all_tok[b], b
        for j in range(steps):
            assert torch.equal(lg[b][j], all_lg[b][j]), (b, j)


def _controlled(lg, counts, bias, presence, frequency):
    x = lg + bias
    hit = counts > 0
    x[hit] = (x[hit] - counts[hit].astype(np.float32) * np.float32(frequency)) - np.float32(presence)
    return x


@pytest.mark.parametrize("V", [32003, 151936])
def test_per_row_sampler_matches_host(V):
    from distributed_llama_b200 import host
    from distributed_llama_b200.ops import cuda_lib as cl
    lib, H = cl.lib(), host()
    rs = np.random.RandomState(V)
    B, launches = 8, 24
    params = np.array([[0.0, 0.9, 0.0, 0.0], [0.8, 0.9, 0.5, 1.0], [1.3, 0.0, -0.5, 0.25], [0.0, 0.5, 1.5, -1.0],
                       [0.7, 0.95, 0.0, 0.0], [1.0, 0.0, 2.0, 2.0], [0.8, 0.7, -2.0, 0.0], [1.1, 0.9, 0.0, -2.0]], dtype=np.float32)
    bias = np.zeros((B, V), dtype=np.float32)
    for b in range(1, B, 2):
        bias[b, rs.choice(V, 50, replace=False)] = rs.uniform(-100, 100, 50).astype(np.float32)
    counts = np.zeros((B, V), dtype=np.uint32)
    seeds = [int(s) for s in rs.randint(1, 2 ** 62, B)]
    rng = torch.tensor(seeds, dtype=torch.int64, device="cuda")
    hs = [H.Sampler(V, float(params[b, 0]), float(params[b, 1]), seeds[b]) for b in range(B)]
    cnt_d = torch.zeros(B, V, dtype=torch.int32, device="cuda")
    bias_d, par_d = torch.from_numpy(bias).cuda(), torch.from_numpy(params).cuda()
    probs = torch.empty(B * V + 16, device="cuda")
    tok = torch.zeros(B, dtype=torch.int32, device="cuda")
    agree = total = 0
    for k in range(launches):
        mask = 0b01000010 if k % 3 == 2 else 0
        lg = (rs.randn(B, V) * 3).astype(np.float32)
        assert lib.dl_sample_rows_per_row(torch.from_numpy(lg).cuda().data_ptr(), V, probs.data_ptr(), V, par_d.data_ptr(), rng.data_ptr(),
                                          tok.data_ptr(), B, mask, bias_d.data_ptr(), V, cnt_d.data_ptr(), V, cl.stream_ptr()) == 0
        got = tok.tolist()
        for b in range(B):
            if (mask >> b) & 1:
                continue
            x = _controlled(lg[b], counts[b], bias[b], params[b, 2], params[b, 3])
            want = int(hs[b].sample(x))
            if params[b, 0] == 0:
                assert want == got[b], (k, b)
            total += 1
            agree += want == got[b]
            counts[b, got[b]] += 1                         # the device counts what it drew
        assert np.array_equal(cnt_d.cpu().numpy().view(np.uint32), counts)
    assert agree >= total - 1, (agree, total)              # the bound of tests/test_gpu_sampling_controls.py


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
        return json.loads(c.getresponse().read())["choices"][0]["message"]["content"]
    finally:
        c.close()


@pytest.mark.parametrize("server", ["python", "native"])
def test_api_parallel_end_to_end(tmp_models, server):
    """dllama-api / dllama-api-native --parallel 4: four concurrent greedy requests return the text each returns alone."""
    m, t = tmp_models["tiny-llama31"]
    port = _free_port()
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = ([sys.executable, "-m", "distributed_llama_b200.apps.api_server"] if server == "python"
           else [os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")])
    proc = subprocess.Popen(cmd + ["--model", m, "--tokenizer", t, "--port", str(port), "--host", "127.0.0.1", "--parallel", "4",
                                   "--temperature", "0"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.5).close()
                break
            except OSError:
                assert proc.poll() is None, proc.stdout.read()
                time.sleep(0.2)
        bodies = [{"messages": [{"role": "user", "content": f"question number {i} " * (i + 1)}], "max_tokens": 24, "temperature": 0}
                  for i in range(4)]
        alone = [_post(port, b) for b in bodies]
        together = [None] * 4

        def go(i):
            together[i] = _post(port, bodies[i])
        ths = [threading.Thread(target=go, args=(i,)) for i in range(4)]
        for th in ths:
            th.start()
        for th in ths:
            th.join(timeout=120)
        assert together == alone
        assert all(a for a in alone)
    finally:
        proc.kill()
        proc.communicate()
