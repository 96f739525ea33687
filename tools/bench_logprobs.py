"""Cost of per-token log-probabilities (csrc/cuda/logprobs.cu) on the synthetic q40 model of bench.py, one GPU, arms alternated.

    python tools/bench_logprobs.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3]

Every measurement runs its arms in turn (off, k = 0, k = 5, k = 20, off, ...) after one untimed run of each and reports the median
(and range) of `--repeats` runs per arm. A step is what InferenceSession.next_token does: upload (token, position), the step,
the logprobs launch and its copy when asked, the 4-byte token copy, one synchronise.
* single-sequence greedy decode (persistent kernel, CUDA-graph replay) from position 2048;
* the same with temperature 0.8 / top-p 0.9 on the device sampler;
* the 8-slot `--parallel` step after 2048-token prompts, every slot greedy, off against k = 20 on every slot;
* CUDA-event device time of the kernel alone at V = 128256 and 151936 for 1 and 8 rows, k = 0 and 20 (median of 3 windows of
  200 launches).
It prints one JSON line per measurement with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = (None, 0, 5, 20)


def name(k):
    return "off" if k is None else f"k{k}"


def alternate(fns, repeats):
    for f in fns.values():
        f()
    ts = {a: [] for a in fns}
    for _ in range(repeats):
        for a, f in fns.items():
            ts[a].append(f())
    return {a: sorted(v) for a, v in ts.items()}


def single_time(eng, start, tokens, k, sampled):
    import torch
    pin_in = torch.zeros(2, dtype=torch.int32).pin_memory()
    pin_out = torch.zeros(1, dtype=torch.int32).pin_memory()
    tok = 7
    if sampled:
        eng.seed_sampler(1234)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(tokens):
        if sampled:
            eng.step_sampled(tok, start + i, 0.8, 0.9)
        else:
            pin_in[0], pin_in[1] = tok, start + i
            eng.tokens[:1].copy_(pin_in[:1], non_blocking=True)
            eng.pos[:1].copy_(pin_in[1:2], non_blocking=True)
            eng.run_decode_step()
        if k is not None:
            eng.logprobs([k], controlled=sampled)
        pin_out.copy_(eng.tokens[:1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        if k is not None:
            eng.read_logprobs()
        tok = int(pin_out[0])
    dt = time.perf_counter() - t0
    assert sampled or eng.mega_active
    return dt


def slots_time(eng, prompts, tokens, k):
    import torch
    n = len(prompts)
    for b in range(n):
        eng.slot_logprobs(b, k)
    tok = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(tokens):
        out, _ = eng.slots_step_logprobs(tok, pos, [True] * n)
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


def kernel_times():
    import torch
    from distributed_llama_b200.runtime.engine import logprobs_rows
    res = {}
    for V in (128256, 151936):
        x = torch.randn(8, V, device="cuda") * 4
        chosen = torch.randint(0, V, (8,), dtype=torch.int32, device="cuda")
        for B in (1, 8):
            for k in (0, 20):
                res[f"V{V}_rows{B}_k{k}"] = event_us(lambda: logprobs_rows(x[:B], chosen[:B], [k] * B))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3.1-8b")
    ap.add_argument("--tokens", type=int, default=64, help="generated tokens per measurement")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from bench import ensure_model
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    from tools.bench_parallel import gpu_info, prompts
    assert torch.cuda.is_available(), "bench_logprobs needs a GPU"
    seq = 8 * (2048 + args.tokens + 1)
    m, _ = ensure_model(args.model)
    w = load_device_weights(ModelFile(m, seq))
    eng = Engine(w, seq_len=seq)
    gpu = gpu_info()
    for sampled in (False, True):
        ts = alternate({k: (lambda k=k: single_time(eng, 2048, args.tokens, k, sampled)) for k in ARMS}, args.repeats)
        row = {name(k): round(args.tokens / ts[k][len(ts[k]) // 2], 1) for k in ARMS}
        print(json.dumps({"gpu": gpu, "measure": "single_sequence_" + ("sampled" if sampled else "greedy"), "start_pos": 2048,
                          "tok_s": row, "tok_s_min_max": {name(k): [round(args.tokens / ts[k][-1], 1), round(args.tokens / ts[k][0], 1)]
                                                          for k in ARMS},
                          "k20_vs_off": round(row["k20"] / row["off"], 4)}), flush=True)
    ps = prompts(8, 2048)
    eng.set_slots(8)
    for b in range(8):
        eng.slot_prefill(b, ps[b][:-1], 0)
        eng.slot_sampling(b, 1000 + b, 0.0, 0.9)
    arms = (None, 20)
    ts = alternate({k: (lambda k=k: slots_time(eng, ps, args.tokens, k)) for k in arms}, args.repeats)
    row = {name(k): round(8 * args.tokens / ts[k][len(ts[k]) // 2], 1) for k in arms}
    print(json.dumps({"gpu": gpu, "measure": "slots_step", "slots": 8, "prompt_len": 2048, "tok_s": row,
                      "ms_per_step": {name(k): round(1000 * ts[k][len(ts[k]) // 2] / args.tokens, 3) for k in arms},
                      "k20_vs_off": round(row["k20"] / row["off"], 4)}), flush=True)
    print(json.dumps({"gpu": gpu, "measure": "kernel_us", "us": kernel_times()}), flush=True)


if __name__ == "__main__":
    main()
