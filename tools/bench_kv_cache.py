"""bf16 against q80 KV cache (`--kv-cache-float-type`) on the synthetic q40 model of bench.py, one GPU, the two arms alternated.

    python tools/bench_kv_cache.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3]

Two engines share one copy of the weights, one per cache type. Every measurement runs bf16, q80, bf16, q80, ... and reports the
median (and range) of `--repeats` runs per arm after one untimed run of each:
* single-sequence greedy decode (persistent kernel, CUDA-graph replay) of `--tokens` tokens starting at positions 2048, 8192 and
  32768. The cache rows before the start are never written: attention reads them all the same, and its time does not depend
  on their values;
* the 8-slot `--parallel` step, every slot busy after a 2048-token prompt;
* CUDA-event device times (median of 3 windows of 200 launches) of slotAttnKernel at 8 rows x 2048 positions and of prefill
  attention on the tensor cores at T = 64 and T = 192 (p0 = 0), with the model's attention shape.
It prints one JSON line per measurement with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = ("bf16", "q80")


def alternate(fns, repeats):
    """fns: arm -> callable returning seconds. One untimed run each, then `repeats` rounds of every arm in turn."""
    for a in ARMS:
        fns[a]()
    ts = {a: [] for a in ARMS}
    for _ in range(repeats):
        for a in ARMS:
            ts[a].append(fns[a]())
    return {a: sorted(v) for a, v in ts.items()}


def decode_time(eng, start, tokens):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = eng.decode_greedy(7, start, tokens)
    torch.cuda.synchronize()
    assert len(out) == tokens and eng.mega_active
    return time.perf_counter() - t0


def slots_time(eng, prompts, tokens):
    import torch
    n = len(prompts)
    tok = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(tokens):
        out = eng.slots_step(tok, pos, [True] * n)
        for b in range(n):
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


def kernel_times(w, n_splits):
    """slotAttnKernel at 8 x 2048 and prefill attention at T = 64 / 192, both cache types, alternated window by window."""
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    lib, sp = cl.lib(), cl.stream_ptr()
    h = w.header
    hd, n_heads, n_kv = h.head_dim, w.n_heads, w.n_kv_heads
    q_dim = n_heads * hd
    stride = q_dim + 2 * n_kv * hd
    B, L = 8, 2048
    qkv = torch.randn(B, stride, device="cuda")
    kf = torch.randn(B, n_kv, L, hd, device="cuda") * 0.1
    vf = torch.randn(B, n_kv, L, hd, device="cuda")
    kb, vb = kf.bfloat16(), vf.bfloat16()

    def q80(x):
        g = x.reshape(-1, 32)
        d = g.abs().amax(dim=1, keepdim=True) / 127.0
        q = torch.round(g / d).to(torch.int8).reshape(x.shape)
        s = torch.zeros(d.numel() + 8, dtype=torch.float16, device="cuda")
        s[:d.numel()] = d.reshape(-1).half()
        return q, s
    (kq, ks), (vq, vs) = q80(kf), q80(vf)
    pos = torch.full((B,), L - 1, dtype=torch.int32, device="cuda")
    partial = torch.empty(B * n_heads * n_splits * (hd + 2), device="cuda")
    counters = torch.zeros(B * n_heads, dtype=torch.int32, device="cuda")
    out = torch.empty(B, q_dim, device="cuda")
    fns = {
        "bf16": lambda: cl.check(lib.dl_slot_attn(qkv.data_ptr(), stride, pos.data_ptr(), kb.data_ptr(), vb.data_ptr(), n_heads, n_kv, hd, L,
                                                  n_splits, B, 0, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, sp), "slot"),
        "q80": lambda: cl.check(lib.dl_slot_attn_q80(qkv.data_ptr(), stride, pos.data_ptr(), kq.data_ptr(), vq.data_ptr(), ks.data_ptr(),
                                                     vs.data_ptr(), n_heads, n_kv, hd, L, n_splits, B, 0, partial.data_ptr(),
                                                     counters.data_ptr(), out.data_ptr(), q_dim, sp), "slot_q80"),
    }
    res = {"slotAttnKernel_8x2048": {a: [] for a in ARMS}}
    for _ in range(3):
        for a in ARMS:
            res["slotAttnKernel_8x2048"][a].append(event_us(fns[a], windows=1))
    # prefill attention: slot 0's cache, the first T rows, T query tokens at p0 = 0
    pq = torch.randn(192, stride, device="cuda")
    pout = torch.empty(192, q_dim, dtype=torch.bfloat16, device="cuda")
    for T in (64, 192):
        key = f"attnPrefillTc_T{T}"
        res[key] = {a: [] for a in ARMS}
        pf = {
            "bf16": lambda T=T: cl.check(lib.dl_attn_prefill_tc(pq.data_ptr(), stride, T, 0, n_heads, n_kv, hd, L, kb.data_ptr(), vb.data_ptr(),
                                                                pout.data_ptr(), q_dim, sp), "prefill"),
            "q80": lambda T=T: cl.check(lib.dl_attn_prefill_tc_q80(pq.data_ptr(), stride, T, 0, n_heads, n_kv, hd, L, kq.data_ptr(),
                                                                   vq.data_ptr(), ks.data_ptr(), vs.data_ptr(), pout.data_ptr(), q_dim, sp),
                                        "prefill_q80"),
        }
        for _ in range(3):
            for a in ARMS:
                res[key][a].append(event_us(pf[a], windows=1))
    return {k: {a: sorted(v)[1] for a, v in d.items()} for k, d in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3.1-8b")
    ap.add_argument("--tokens", type=int, default=64, help="generated tokens per measurement")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--positions", default="2048,8192,32768")
    args = ap.parse_args()
    import torch
    from bench import ensure_model
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    from tools.bench_parallel import gpu_info, prompts
    assert torch.cuda.is_available(), "bench_kv_cache needs a GPU"
    positions = [int(x) for x in args.positions.split(",")]
    seq = max(max(positions) + args.tokens + 1, 8 * (2048 + args.tokens + 1))
    m, _ = ensure_model(args.model)
    w = load_device_weights(ModelFile(m, seq))
    engs = {a: Engine(w, seq_len=seq, kv_cache_float_type=a) for a in ARMS}
    gpu = gpu_info()
    for p in positions:
        ts = alternate({a: (lambda e=engs[a]: decode_time(e, p, args.tokens)) for a in ARMS}, args.repeats)
        row = {a: round(args.tokens / ts[a][len(ts[a]) // 2], 1) for a in ARMS}
        print(json.dumps({"gpu": gpu, "measure": "single_sequence_greedy", "start_pos": p, "tok_s": row,
                          "tok_s_min_max": {a: [round(args.tokens / ts[a][-1], 1), round(args.tokens / ts[a][0], 1)] for a in ARMS},
                          "q80_vs_bf16": round(row["q80"] / row["bf16"], 3)}), flush=True)
    ps = prompts(8, 2048)
    for a in ARMS:
        engs[a].set_slots(8)
        for b in range(8):
            engs[a].slot_prefill(b, ps[b][:-1], 0)
            engs[a].slot_sampling(b, 1000 + b, 0.0, 0.9)
    ts = alternate({a: (lambda e=engs[a]: slots_time(e, ps, args.tokens)) for a in ARMS}, args.repeats)
    row = {a: round(8 * args.tokens / ts[a][len(ts[a]) // 2], 1) for a in ARMS}
    print(json.dumps({"gpu": gpu, "measure": "slots_step", "slots": 8, "prompt_len": 2048, "tok_s": row,
                      "ms_per_step": {a: round(1000 * ts[a][len(ts[a]) // 2] / args.tokens, 3) for a in ARMS},
                      "q80_vs_bf16": round(row["q80"] / row["bf16"], 3)}), flush=True)
    h = w.header
    kv_bytes = {a: int(2 * 8 * w.n_kv_heads * 2048 * h.head_dim * (2 if a == "bf16" else 34 / 32)) for a in ARMS}
    print(json.dumps({"gpu": gpu, "measure": "kernels_us", "us": kernel_times(w, engs["bf16"].n_splits),
                      "slot_kv_bytes_per_layer": kv_bytes}), flush=True)


if __name__ == "__main__":
    main()
