"""Cost of the paged KV-cache slot layout (`--parallel-cache paged`) against the split one, in one process, arms alternated.

    python tools/bench_paged_slots.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3]

On the synthetic q40 model of bench.py, one GPU, 8 slots with every slot busy. For prompts of 64 and 2048 tokens, greedy and
sampled (temperature 0.8, top-p 0.9), it times the 8-slot step in three arms, alternated: split, paged with each slot's pages
contiguous, and paged with the slots' pages interleaved (reserved one page at a time, round robin). A paged row reserves its
next page inside the timed loop, as the server does. Each figure is the median of `--repeats` runs after one untimed warm-up, a
host clock around work that ends in a device synchronise. Then the device time (CUDA events, median of 3 windows of 200
launches) of slotAttnKernel over 8 rows at position 2047 in the three layouts, and of a 2048-token slot prefill in both
layouts. One JSON line per measurement; the GPU name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, PAGE = 8, 64
ARMS = ("split", "paged", "scattered")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def prompts(plen):
    return [[(7 * i + 3 + 101 * b) % 1000 + 1 for i in range(plen)] for b in range(N)]


def setup(eng, arm, rows):
    eng.set_slots(N, "split" if arm == "split" else "paged")
    if arm == "paged":
        for b in range(N):
            assert eng.slot_reserve(b, rows)
    elif arm == "scattered":
        for r in range(PAGE, rows + PAGE, PAGE):
            for b in range(N):
                assert eng.slot_reserve(b, min(r, rows))


def time_step(eng, arm, plen, tokens, T):
    import torch
    ps = prompts(plen)
    setup(eng, arm, plen)
    for b in range(N):
        eng.slot_prefill(b, ps[b][:-1], 0)
        eng.slot_sampling(b, 1000 + b, T, 0.9)
    tok = [p[-1] for p in ps]
    pos = [plen - 1] * N
    active = [True] * N
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(tokens):
        if arm != "split":
            for b in range(N):
                assert eng.slot_reserve(b, pos[b] + 1)
        out = eng.slots_step(tok, pos, active)
        for b in range(N):
            tok[b], pos[b] = out[b], pos[b] + 1
    return time.perf_counter() - t0


def event_us(fn, windows=3, launches=200):
    import torch
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
    return round(sorted(ts)[len(ts) // 2], 2)


def time_attention(eng, p=2047):
    """slotAttnKernel over N rows at position p: split slots, paged contiguous and paged interleaved pages."""
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    w, h = eng.w, eng.w.header
    hd, n_heads, n_kv = h.head_dim, w.n_heads, w.n_kv_heads
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    L = p + 1
    per = -(-L // PAGE)
    rows = N * per * PAGE
    qkv = torch.randn(N, q_dim + 2 * kv_dim, device="cuda")
    kc = (torch.randn(n_kv, rows, hd, device="cuda") * 0.1).bfloat16()
    vc = torch.randn(n_kv, rows, hd, device="cuda").bfloat16()
    pos = torch.full((N,), p, dtype=torch.int32, device="cuda")
    partial = torch.empty(N * n_heads * eng.n_splits * (hd + 2), device="cuda")
    counters = torch.zeros(N * n_heads, dtype=torch.int32, device="cuda")
    out = torch.empty(N, q_dim, device="cuda")
    contiguous = torch.arange(N * per, dtype=torch.int32, device="cuda").view(N, per)
    interleaved = torch.arange(N * per, dtype=torch.int32, device="cuda").view(per, N).t().contiguous()
    lib, sp, stride = cl.lib(), cl.stream_ptr(), q_dim + 2 * kv_dim

    def split():
        cl.check(lib.dl_slot_attn(qkv.data_ptr(), stride, pos.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_heads, n_kv, hd, per * PAGE,
                                  eng.n_splits, N, 0, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, sp), "dl_slot_attn")

    def paged(table):
        return lambda: cl.check(lib.dl_slot_attn_paged(qkv.data_ptr(), stride, pos.data_ptr(), kc.data_ptr(), vc.data_ptr(), None, None,
                                                       table.data_ptr(), per, rows, n_heads, n_kv, hd, per * PAGE, eng.n_splits, N, 0,
                                                       partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, sp),
                                "dl_slot_attn_paged")
    res = {arm: [] for arm in ARMS}
    for _ in range(3):   # alternated
        for arm, fn in (("split", split), ("paged", paged(contiguous)), ("scattered", paged(interleaved))):
            res[arm].append(event_us(fn))
    return {arm: sorted(v)[1] for arm, v in res.items()}


def time_prefill(eng, plen=2048, repeats=5):
    """Device time of one plen-token slot prefill into slot 0, split and paged (interleaved pages), alternated; milliseconds."""
    import torch
    ps = prompts(plen + 1)[0]
    res = {"split": [], "scattered": []}
    for _ in range(repeats):
        for arm in res:
            setup(eng, arm, plen)
            eng.slot_prefill(0, ps[:plen], 0)   # warm-up of the shape
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.slot_prefill(0, ps[:plen], 0)
            b.record()
            torch.cuda.synchronize()
            res[arm].append(a.elapsed_time(b))
    return {arm: round(sorted(v)[len(v) // 2], 3) for arm, v in res.items()}


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
    assert torch.cuda.is_available(), "bench_paged_slots needs a GPU"
    plens = [int(x) for x in args.prompt_lens.split(",")]
    seq = N * (max(plens) + args.tokens + PAGE)
    m, t = ensure_model(args.model)
    sess = InferenceSession(m, t, max_seq_len=seq, temperature=0.8, topp=0.9, seed=1234)
    eng = sess.engine
    gpu = gpu_info()
    for plen in plens:
        for T in (0.8, 0.0):
            times = {arm: [] for arm in ARMS}
            for arm in ARMS:   # warm-up of every arm
                time_step(eng, arm, plen, args.tokens, T)
            for _ in range(args.repeats):
                for arm in ARMS:
                    times[arm].append(time_step(eng, arm, plen, args.tokens, T))
            med = {arm: sorted(v)[len(v) // 2] for arm, v in times.items()}
            print(json.dumps({"gpu": gpu, "prompt_len": plen, "temperature": T, "n_slots": N,
                              "ms_per_step": {arm: round(1000 * med[arm] / args.tokens, 3) for arm in ARMS},
                              "paged_vs_split": round(med["paged"] / med["split"], 4),
                              "scattered_vs_split": round(med["scattered"] / med["split"], 4)}), flush=True)
    print(json.dumps({"gpu": gpu, "slotAttnKernel_us": time_attention(eng), "rows": N, "position": 2047}), flush=True)
    print(json.dumps({"gpu": gpu, "slot_prefill_ms": time_prefill(eng), "tokens": 2048}), flush=True)


if __name__ == "__main__":
    main()
