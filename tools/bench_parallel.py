"""Throughput of independent sequences decoded together in KV-cache slots (`dllama-api --parallel N`) against the single-sequence path.

    python tools/bench_parallel.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3]

On the synthetic q40 model of bench.py, one GPU. For every prompt length (64 and 2048 tokens) and sampling mode (temperature
0.8 / top-p 0.9, and greedy) it measures:
* N = 1 on the single-sequence path (`--parallel 1`: persistent decode kernel, graph replay when greedy), token by token as the
  server runs it;
* N = 2, 4, 8 slots with every slot busy, each with its own prompt, one batched step per token;
* 8 slots with 1 and 4 busy: the cost of always running the padded power-of-two batch when few requests are in flight.
Each figure is the median of `--repeats` runs after one untimed warm-up run of the same shape, timed with a host clock around
work that ends in a device synchronise (every step reads its tokens back). It prints one JSON line per measurement: aggregate
generated tokens/s and milliseconds per step. Then the device time (CUDA events, median of 3 windows of 200 launches) of
slotAttnKernel for 8 rows at position 2047 against attnDecodeKernel over the same 8 sequences (one launch per sequence: each
has its own cache) with the model's attention shape. The GPU name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAX_N = 8


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def prompts(n, plen):
    return [[(7 * i + 3 + 101 * b) % 1000 + 1 for i in range(plen)] for b in range(n)]


def time_single(sess, prompt, tokens, T):
    """N = 1: the server's single-completion loop (api.run_choices) on the unsplit engine."""
    import torch
    from distributed_llama_b200.api import run_choices
    sess.engine.set_slots(1)
    sess.sampler.set_temperature(T)
    sess.engine.prefill(prompt[:-1], 0, want_logits=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run_choices(sess, prompt[-1], len(prompt) - 1, 1, tokens, sess.engine.seq_len, sess.sampler, 1234, lambda i, t: False)
    dt = time.perf_counter() - t0
    assert len(out[0]) == tokens
    return dt


def time_slots(eng, n_slots, busy, plen, tokens, T):
    """`busy` of `n_slots` slots decode `tokens` tokens each, one slots step per token."""
    import torch
    eng.set_slots(n_slots)
    ps = prompts(busy, plen)
    for b in range(busy):
        eng.slot_prefill(b, ps[b][:-1], 0)
        eng.slot_sampling(b, 1000 + b, T, 0.9)
    active = [b < busy for b in range(n_slots)]
    tok = [ps[b][-1] if b < busy else 0 for b in range(n_slots)]
    pos = [plen - 1 if b < busy else 0 for b in range(n_slots)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(tokens):
        out = eng.slots_step(tok, pos, active)
        for b in range(busy):
            tok[b], pos[b] = out[b], pos[b] + 1
    return time.perf_counter() - t0


def median_of(fn, repeats):
    fn()                                     # warm-up of the same shape
    ts = sorted(fn() for _ in range(repeats))
    return ts[len(ts) // 2], ts[0], ts[-1]


def time_attention(eng, B=8, p=2047, windows=3, launches=200):
    """slotAttnKernel over B slots against attnDecodeKernel over the same B sequences (one launch each), in microseconds."""
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    w, h = eng.w, eng.w.header
    hd, n_heads, n_kv = h.head_dim, w.n_heads, w.n_kv_heads
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    L = p + 1
    qkv = torch.randn(B, q_dim + 2 * kv_dim, device="cuda")
    kc = (torch.randn(B, n_kv, L, hd, device="cuda") * 0.1).bfloat16()
    vc = torch.randn(B, n_kv, L, hd, device="cuda").bfloat16()
    pos = torch.full((B,), p, dtype=torch.int32, device="cuda")
    partial = torch.empty(B * n_heads * eng.n_splits * (hd + 2), device="cuda")
    counters = torch.zeros(B * n_heads, dtype=torch.int32, device="cuda")
    out = torch.empty(B, q_dim, device="cuda")
    lib, sp = cl.lib(), cl.stream_ptr()
    stride = q_dim + 2 * kv_dim

    def slots():
        cl.check(lib.dl_slot_attn(qkv.data_ptr(), stride, pos.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_heads, n_kv, hd, L, eng.n_splits,
                                  B, 0, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, sp), "dl_slot_attn")

    def decode():
        for b in range(B):
            cl.check(lib.dl_attn_decode(qkv[b].data_ptr(), stride, pos[b:].data_ptr(), kc[b].data_ptr(), vc[b].data_ptr(), n_heads, n_kv, hd,
                                        L, eng.n_splits, partial.data_ptr(), counters.data_ptr(), out[b].data_ptr(), q_dim, None, 1, sp),
                     "dl_attn_decode")

    res = {}
    for name, fn in (("slotAttnKernel", slots), ("attnDecodeKernel", decode)):
        for _ in range(20):
            fn()
        ts = []
        for _ in range(windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(launches):
                fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1000.0 / launches)
        res[name] = round(sorted(ts)[len(ts) // 2], 2)
    kv_bytes = 2 * B * n_kv * L * hd * 2   # K and V of every sequence, bf16
    return res, kv_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3.1-8b")
    ap.add_argument("--tokens", type=int, default=64, help="generated tokens per sequence")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--prompt-lens", default="64,2048")
    args = ap.parse_args()
    import torch
    from bench import ensure_model
    from distributed_llama_b200.api import InferenceSession
    assert torch.cuda.is_available(), "bench_parallel needs a GPU"
    plens = [int(x) for x in args.prompt_lens.split(",")]
    seq = MAX_N * (max(plens) + args.tokens + 1)
    m, t = ensure_model(args.model)
    sess = InferenceSession(m, t, max_seq_len=seq, temperature=0.8, topp=0.9, seed=1234)
    eng = sess.engine
    gpu = gpu_info()
    for plen in plens:
        for T in (0.8, 0.0):
            base, lo, hi = median_of(lambda: time_single(sess, prompts(1, plen)[0], args.tokens, T), args.repeats)
            print(json.dumps({"gpu": gpu, "prompt_len": plen, "temperature": T, "path": "single", "n_slots": 1, "busy": 1,
                              "tok_s": round(args.tokens / base, 1), "ms_per_step": round(1000 * base / args.tokens, 3),
                              "tok_s_min_max": [round(args.tokens / hi, 1), round(args.tokens / lo, 1)]}), flush=True)
            for n_slots, busy in ((2, 2), (4, 4), (8, 8), (8, 1), (8, 4)):
                dt, lo, hi = median_of(lambda: time_slots(eng, n_slots, busy, plen, args.tokens, T), args.repeats)
                print(json.dumps({"gpu": gpu, "prompt_len": plen, "temperature": T, "path": "slots", "n_slots": n_slots, "busy": busy,
                                  "tok_s": round(busy * args.tokens / dt, 1), "ms_per_step": round(1000 * dt / args.tokens, 3),
                                  "tok_s_min_max": [round(busy * args.tokens / hi, 1), round(busy * args.tokens / lo, 1)],
                                  "vs_single": round((busy * args.tokens / dt) / (args.tokens / base), 2)}), flush=True)
    eng.set_slots(1)
    us, kv_bytes = time_attention(eng)
    print(json.dumps({"gpu": gpu, "kernels_us": us, "rows": 8, "position": 2047, "kv_bytes_per_layer": kv_bytes}), flush=True)


if __name__ == "__main__":
    main()
