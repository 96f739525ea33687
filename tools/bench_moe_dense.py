"""Qwen3-30B-A3B decode with f16 expert matrices (the dense-weight MoE path) beside the q40 preset, one GPU, in one run.

    python tools/bench_moe_dense.py [--steps 64] [--repeats 3] [--max-seq-len 2048]

Both models are random-init device weights in the loader's layout (models/loader.py synthetic_device_weights): a 61 GB f16 file
would take far longer to write than to run. The q40 model is measured first and freed before the f16 one is built. For each:
* greedy decode (CUDA-graph replay) of `--steps` tokens after a 64-token prompt, median of `--repeats` windows after one untimed
  window: tokens/s, ms/token, the bytes a token streams (attention matrices, router gates, the k active experts of every layer,
  the logits matrix; computed from the device tensors) and those bytes over the step time;
* f16 only: CUDA-event times of the MoE feed-forward of one layer (router + W1|W3 + W2, `dl_moe_decode_ffn_dense`) and of the
  router alone (`dl_moe_router`), each the median of 3 windows of 200 launches, and the two expert kernels' share of the FFN from
  a torch.profiler run of its own.
Each line is JSON; the first one carries the GPU name and power limit read in the same run.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, clk = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def nbytes(t):
    return 0 if t is None else t.numel() * t.element_size()


def token_bytes(W):
    """Weight bytes one decode step streams: every attention matrix, the router gates, k of the local experts, the logits matrix."""
    h = W.header
    k = h.n_active_experts
    total = nbytes(W.wcls.qs) + nbytes(W.wcls.scales) + nbytes(W.final_norm) + h.dim * 4
    for L in W.layers:
        total += nbytes(L.qkv.qs) + nbytes(L.qkv.scales) + nbytes(L.wo.qs) + nbytes(L.wo.scales) + nbytes(L.moe_gate)
        expert = (nbytes(L.w13.qs) + nbytes(L.w13.scales) + nbytes(L.w2.qs) + nbytes(L.w2.scales)) // W.n_local_experts
        total += k * expert + nbytes(L.norm0) + nbytes(L.norm1)
    return total


def decode_rate(eng, steps, repeats):
    import torch
    prompt = [(7 * i + 3) % 1000 + 1 for i in range(64)]
    eng.prefill(prompt[:-1], 0, want_logits=False)
    p0 = len(prompt) - 1
    eng.decode_greedy(prompt[-1], p0, steps)      # warm-up, graph capture
    times = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        eng.decode_greedy(prompt[-1], p0, steps)
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) / steps)
    return statistics.median(times), times


def measure(weight_type, args, cfg):
    import torch
    from distributed_llama_b200.models.loader import synthetic_device_weights
    from distributed_llama_b200.runtime import Engine
    t0 = time.time()
    W = synthetic_device_weights(cfg, max_seq_len=args.max_seq_len, weight_type=weight_type)
    eng = Engine(W)
    load_s = time.time() - t0
    ms, all_ms = decode_rate(eng, args.steps, args.repeats)
    b = token_bytes(W)
    row = {"model": cfg.name, "weights": weight_type, "decode_tok_s": round(1000.0 / ms, 2), "ms_per_token": round(ms, 4),
           "ms_per_token_windows": [round(x, 4) for x in all_ms], "bytes_per_token": b,
           "achieved_TB_s": round(b / (ms * 1e-3) / 1e12, 3), "device_GB": round(torch.cuda.memory_allocated() / 1e9, 2),
           "build_s": round(load_s, 1), "steps": args.steps}
    print(json.dumps(row), flush=True)
    if weight_type != "q40":
        print(json.dumps(ffn_times(eng, W, weight_type)), flush=True)
    del eng, W
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def ffn_times(eng, W, weight_type):
    """CUDA-event times of one layer's MoE feed-forward and of its router; the expert kernels' split from torch.profiler."""
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    h = W.header
    L = W.layers[0]
    dim, ff, E, k = h.dim, W.ff_dim, h.n_experts, h.n_active_experts
    wt = 1 if weight_type == "f32" else 2
    sms = eng.num_sms
    f32 = dict(device="cuda", dtype=torch.float32)
    x = torch.randn(dim, **f32)
    out = torch.zeros(dim, **f32)
    logits, wts = torch.zeros(E, **f32), torch.zeros(k, **f32)
    counter, ids = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(k, dtype=torch.int32, device="cuda")
    hb, scratch = torch.zeros(k, ff, **f32), torch.zeros(k, dim, **f32)
    counters = torch.zeros(max(1, sms // k), dtype=torch.int32, device="cuda")
    lib, sp = cl.lib(), cl.stream_ptr()

    def ffn():
        cl.check(lib.dl_moe_decode_ffn_dense(wt, x.data_ptr(), out.data_ptr(), L.norm1.data_ptr(), L.moe_gate.data_ptr(), L.w13.qs.data_ptr(),
                                             L.w2.qs.data_ptr(), dim, ff, E, k, W.first_expert, W.n_local_experts, h.norm_epsilon,
                                             logits.data_ptr(), counter.data_ptr(), ids.data_ptr(), wts.data_ptr(), hb.data_ptr(),
                                             scratch.data_ptr(), counters.data_ptr(), sms, 0, sp), "moe_decode_ffn_dense")

    def router():
        cl.check(lib.dl_moe_router(x.data_ptr(), L.norm1.data_ptr(), L.moe_gate.data_ptr(), h.norm_epsilon, dim, E, k, logits.data_ptr(),
                                   counter.data_ptr(), ids.data_ptr(), wts.data_ptr(), 1, sp), "moe_router")

    def event_us(fn, n=200):
        fn()
        res = []
        for _ in range(3):
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(n):
                fn()
            e.record()
            torch.cuda.synchronize()
            res.append(s.elapsed_time(e) * 1000.0 / n)
        return statistics.median(res)

    ffn_us, router_us = event_us(ffn), event_us(router)
    expert_bytes = k * (nbytes(L.w13.qs) + nbytes(L.w2.qs)) // W.n_local_experts
    split = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            ffn()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "gemvDenseMoeKernel" in ev.key:
            kind = "w13_swiglu" if ", 0, 2, " in ev.key or ",0,2," in ev.key.replace(" ", "") else "w2_moe_down"
            split[kind] = {"kernel": ev.key, "us_per_launch": round(ev.device_time_total / max(1, ev.count), 2)}
    return {"weights": weight_type, "ffn_us": round(ffn_us, 2), "router_us": round(router_us, 2),
            "experts_us": round(ffn_us - router_us, 2), "expert_bytes": expert_bytes,
            "experts_TB_s": round(expert_bytes / ((ffn_us - router_us) * 1e-6) / 1e12, 3), "profiler_split": split}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-seq-len", type=int, default=2048)
    ap.add_argument("--model", default="qwen3-30b-a3b")
    ap.add_argument("--weights", default="q40,f16", help="comma-separated weight types, measured in this order")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_moe_dense needs a GPU")
    from distributed_llama_b200.models.config import get_config
    cfg = get_config(args.model)
    print(json.dumps(gpu_info()), flush=True)
    for wt in args.weights.split(","):
        measure(wt, args, cfg)


if __name__ == "__main__":
    main()
