"""Decode tokens/s + TTFT of one of the large BASELINE.json configurations on random-init device weights (no `.m` file is written:
models/loader.py synthetic_device_weights). Run under torchrun for N > 1.

    python tools/bench_config.py qwen3-14b [--pos 0] [--steps 64] [--max-seq-len 4096]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from distributed_llama_b200.models.config import get_config
from distributed_llama_b200.models.loader import synthetic_device_weights
from distributed_llama_b200.runtime import Engine

ap = argparse.ArgumentParser()
ap.add_argument("model")
ap.add_argument("--steps", type=int, default=64)
ap.add_argument("--prompt-len", type=int, default=64)
ap.add_argument("--pos", type=int, default=0, help="start decoding at this position (the KV cache below it holds random rows)")
ap.add_argument("--max-seq-len", type=int, default=2048)
ap.add_argument("--moe-mode", default="auto")
args = ap.parse_args()
world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
comm = None
if world > 1:
    from distributed_llama_b200.parallel.comm import Communicator
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    comm = Communicator()
cfg = get_config(args.model)
t0 = time.time()
W = synthetic_device_weights(cfg, rank, world, f"cuda:{local}", moe_mode=args.moe_mode, max_seq_len=args.max_seq_len)
eng = Engine(W, comm=comm)
load_s = time.time() - t0


def sync():
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def mx(v):
    if world == 1:
        return v
    t = torch.tensor([v], device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


prompt = [(7 * i + 3) % 1000 + 1 for i in range(args.prompt_len)]
ttft = []
for _ in range(3):
    sync()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    eng.prefill(prompt[:-1], 0, want_logits=False)
    eng.decode_greedy(prompt[-1], len(prompt) - 1, 1)
    e.record()
    torch.cuda.synchronize()
    ttft.append(mx(s.elapsed_time(e)))
pos0 = max(args.pos, len(prompt) - 1)
if pos0 > len(prompt) - 1:
    for kc, vc in zip(eng.k_cache, eng.v_cache):       # long-context decode: fill the cache below pos0 with plausible rows
        kc[:, :pos0].normal_(0, 0.5)
        vc[:, :pos0].normal_(0, 0.5)
eng.decode_greedy(prompt[-1], pos0, 8)
sync()
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
eng.decode_greedy(prompt[-1], pos0, args.steps)
e.record()
sync()
ms = mx(s.elapsed_time(e)) / args.steps
if rank == 0:
    wb = sum(L.qkv.qs.numel() * 4 + L.qkv.scales.numel() * 2 + L.wo.qs.numel() * 4 + L.wo.scales.numel() * 2 + L.w13.qs.numel() * 4 +
             L.w13.scales.numel() * 2 + L.w2.qs.numel() * 4 + L.w2.scales.numel() * 2 for L in W.layers) + W.wcls.qs.numel() * 4 + W.wcls.scales.numel() * 2
    h = W.header
    if h.n_experts > 0:      # only the routed experts are streamed per token
        per_layer_moe = sum(L.w13.qs.numel() * 4 + L.w13.scales.numel() * 2 + L.w2.qs.numel() * 4 + L.w2.scales.numel() * 2 for L in W.layers)
        wb = wb - per_layer_moe + per_layer_moe * h.n_active_experts // max(1, W.n_local_experts if W.moe_mode == "tp" else h.n_experts)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm, hbm_source = peaks.get("hbm_gbs"), "measured"
    if not hbm:
        hbm, hbm_source = 3350.0, "H100 SXM data sheet"
    print(json.dumps({"model": args.model, "n_gpus": world, "decode_tok_s": round(1000.0 / ms, 1), "ms_per_step": round(ms, 4), "decode_pos": pos0,
                      "ttft_ms": round(min(ttft[1:]), 3), "prompt_len": args.prompt_len, "decode_path": "persistent megakernel" if (eng.mega and eng.mega_active) else "multi-kernel",
                      "moe_mode": W.moe_mode, "weight_bytes_streamed_per_step_per_gpu": int(wb),
                      "frac_of_peak_hbm": round(wb / ms / 1e6 / hbm, 3), "peak_hbm_gbs": hbm, "peak_hbm_source": hbm_source, "weights_init_s": round(load_s, 1),
                      "data": "random-init device weights (no file), synthetic prompt"}), flush=True)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
