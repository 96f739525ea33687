"""Pipeline timeline of the prefill GEMM (CTA 0): where the MMA warpgroup (warp 4) and one dequant group spend their cycles.
Needs DL_GEMM_DEBUG=512 (set here). Output: per-k-block stamps in SM clocks relative to the first event."""
import ctypes as C, os, sys
os.environ["DL_GEMM_DEBUG"] = str(512 | int(os.environ.get("DL_GEMM_DEBUG", "0")))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from distributed_llama_b200 import ops
from distributed_llama_b200.ops import DeviceQ40, cuda_lib
from tools.microbench_gemm import rand_dev

T = int(sys.argv[1]) if len(sys.argv) > 1 else 64
d, n = 6144, 4096
w = rand_dev(d, n)
act = torch.randn(T, n, device="cuda").bfloat16()
out = torch.zeros(T, d, device="cuda")
flush = torch.ones(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
for _ in range(3):
    _ = flush.view(torch.int64).sum()
    ops.gemm_q40_tc(w, act, epi=ops.GEPI_STORE_F32, out=out, variant="tma")
torch.cuda.synchronize()
buf = (C.c_ulonglong * 4096)()
lib = cuda_lib.lib()
lib.dl_gemm_trace_read.argtypes = [C.c_void_p]
assert lib.dl_gemm_trace_read(buf) == 0
t = np.array(buf[:], dtype=np.int64)
mma = t[:1024].reshape(256, 4)[:64]
dq = t[1024:1024 + 4 * 64 * 8].reshape(4, 64, 8)[:, :16, :6]
t0 = min(mma[0, 0], dq[:, 0, 0].min())
print("MMA warpgroup, per k-block: start  +waitB  +waitA  +issue+release   (period)")
prev = None
for i in range(64):
    s, b, a_, e = mma[i] - t0
    print(f"kb{i:3d} {s:8d} {b - s:6d} {a_ - b:6d} {e - a_:6d}   {'' if prev is None else s - prev}")
    prev = s
for g in range(4):
    print(f"dequant group {g}, per raw chunk: start +waitRaw +lds +waitSlot +convert +fence")
    for i in range(16):
        x = dq[g, i] - t0
        print(f"kq{i:3d} {x[0]:8d} {x[1]-x[0]:6d} {x[2]-x[1]:6d} {x[3]-x[2]:6d} {x[4]-x[3]:6d} {x[5]-x[4]:6d}")
