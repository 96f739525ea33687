"""Cost of the sampling filters top_k / min_p (csrc/cuda/sampler.cu) on the synthetic q40 model of bench.py, one GPU, arms alternated.

    python tools/bench_sampling_filters.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3]

Every measurement runs its arms in turn (off, top_k = 40, min_p = 0.05, both, off, ...) after one untimed run of each and reports
the median (and range) of `--repeats` runs per arm:
* single-sequence sampled decode (temperature 0.8, top-p 0.9) from position 2048: upload, step, device draw, token copy, sync;
* the 8-slot `--parallel` step after 2048-token prompts, every slot sampled, without and with top_k = 40 and min_p = 0.05;
* CUDA-event device time of sampleKernel alone at V = 128256 and 151936, one row, per arm (median of 3 windows of 200 launches).
It prints one JSON line per measurement with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = {"off": (0, 0.0), "top_k40": (40, 0.0), "min_p0.05": (0, 0.05), "both": (40, 0.05)}


def single_time(eng, start, tokens, arm):
    import torch
    eng.set_sampling_filters(*ARMS[arm])
    pin_out = torch.zeros(1, dtype=torch.int32).pin_memory()
    tok = 7
    eng.seed_sampler(1234)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(tokens):
        eng.step_sampled(tok, start + i, 0.8, 0.9)
        pin_out.copy_(eng.tokens[:1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        tok = int(pin_out[0])
    return time.perf_counter() - t0


def slots_time(eng, prompts, tokens, arm):
    import torch
    n = len(prompts)
    for b in range(n):
        k, p = ARMS[arm]
        eng.slot_sampling(b, 1000 + b, 0.8, 0.9, top_k=k, min_p=p)
    tok = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(tokens):
        out = eng.slots_step(tok, pos, [True] * n)
        for b in range(n):
            tok[b], pos[b] = out[b], pos[b] + 1
    return time.perf_counter() - t0


def kernel_times():
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    from tools.bench_logprobs import event_us
    lib = cl.lib()
    res = {}
    for V in (128256, 151936):
        x = torch.randn(V, device="cuda") * 4
        probs = torch.empty(V + 16, device="cuda")
        rng = torch.tensor([99], dtype=torch.int64, device="cuda")
        tok = torch.zeros(1, dtype=torch.int32, device="cuda")
        for arm, (k, p) in ARMS.items():
            res[f"V{V}_{arm}"] = event_us(lambda k=k, p=p: lib.dl_sample_logits_filtered(x.data_ptr(), probs.data_ptr(), V, 0.8, 0.9, k, p,
                                                                                        rng.data_ptr(), tok.data_ptr(), cl.stream_ptr()))
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
    from tools.bench_logprobs import alternate
    from tools.bench_parallel import gpu_info, prompts
    assert torch.cuda.is_available(), "bench_sampling_filters needs a GPU"
    seq = 8 * (2048 + args.tokens + 1)
    m, _ = ensure_model(args.model)
    w = load_device_weights(ModelFile(m, seq))
    eng = Engine(w, seq_len=seq)
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu, "measure": "kernel_us", "us": kernel_times()}), flush=True)
    ts = alternate({a: (lambda a=a: single_time(eng, 2048, args.tokens, a)) for a in ARMS}, args.repeats)
    row = {a: round(args.tokens / ts[a][len(ts[a]) // 2], 1) for a in ARMS}
    print(json.dumps({"gpu": gpu, "measure": "single_sequence_sampled", "start_pos": 2048, "tok_s": row,
                      "tok_s_min_max": {a: [round(args.tokens / ts[a][-1], 1), round(args.tokens / ts[a][0], 1)] for a in ARMS},
                      "ms_per_token": {a: round(1000 * ts[a][len(ts[a]) // 2] / args.tokens, 3) for a in ARMS}}), flush=True)
    eng.set_sampling_filters(0, 0.0)
    ps = prompts(8, 2048)
    eng.set_slots(8)
    for b in range(8):
        eng.slot_prefill(b, ps[b][:-1], 0)
    arms = ("off", "both")
    ts = alternate({a: (lambda a=a: slots_time(eng, ps, args.tokens, a)) for a in arms}, args.repeats)
    row = {a: round(8 * args.tokens / ts[a][len(ts[a]) // 2], 1) for a in arms}
    print(json.dumps({"gpu": gpu, "measure": "slots_step_sampled", "slots": 8, "prompt_len": 2048, "tok_s": row,
                      "ms_per_step": {a: round(1000 * ts[a][len(ts[a]) // 2] / args.tokens, 3) for a in arms}}), flush=True)


if __name__ == "__main__":
    main()
