"""Tensor-core prefill GEMM microbenchmark at Llama-3.1-8B shapes (CUDA events, weights >> L2 between shapes)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from distributed_llama_b200 import ops
from distributed_llama_b200.ops import DeviceQ40

def rand_dev(d, n):
    w = DeviceQ40.empty(d, n)
    w.qs.random_(-2**31, 2**31 - 1)
    w.scales.copy_((torch.rand(d, n // 32, device="cuda") * 0.01).half())
    return w

def bench(name, d, n, T, epi, variant="auto", iters=10):
    w = rand_dev(d, n)
    act = torch.randn(T, n, device="cuda").bfloat16()
    if epi == ops.GEPI_SWIGLU_BF16:
        out = torch.zeros(T, d // 2, device="cuda", dtype=torch.bfloat16)
    else:
        out = torch.zeros(T, d, device="cuda")
    flush = torch.ones(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    evs = []
    for i in range(iters + 2):
        _ = flush.view(torch.int64).sum()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); ops.gemm_q40_tc(w, act, epi=epi, out=out, variant=variant); e.record()
        evs.append((s, e))
    torch.cuda.synchronize()
    us = float(np.median([s.elapsed_time(e) * 1e3 for s, e in evs[2:]]))
    flops = 2.0 * d * n * T
    byts = d * n * 0.5625
    return dict(kernel=name, variant=variant, d=d, n=n, T=T, us=round(us, 1), tflops=round(flops / us / 1e6, 1), weight_gbs=round(byts / us / 1e3, 1))

if __name__ == "__main__":
    T = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    for v in ("tma",):
        for name, d, n, epi in (("qkv", 6144, 4096, ops.GEPI_STORE_F32), ("wo", 4096, 4096, ops.GEPI_RESIDUAL),
                                ("w13", 28672, 4096, ops.GEPI_SWIGLU_BF16), ("w2", 4096, 14336, ops.GEPI_RESIDUAL)):
            print(json.dumps(bench(name, d, n, T, epi, v)), flush=True)
