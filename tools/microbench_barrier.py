"""Times the software grid-barrier candidates of csrc/cuda/bench_barrier.cu (one CTA per SM, 1000 barriers each)."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from distributed_llama_b200.ops import cuda_lib as cl

lib = cl.lib()
lib.dl_bench_grid_barrier.argtypes = [C.c_int, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                      C.c_int, C.c_void_p]
lib.dl_bench_grid_barrier.restype = C.c_int
sms = torch.cuda.get_device_properties(0).multi_processor_count
stream_buf = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
names = {0: "red.release + ld.acquire poll (shipped)", 1: "relaxed red/poll, no fence (lower bound, not a data barrier)",
         2: "per-CTA flag lines, warp polls one line per CTA", 3: "8 group counters, 8 pollers", 4: "fence + relaxed red, relaxed polls + fence",
         5: "flag words in one array, warp polls with 16-byte loads"}
iters = 1000
for traffic in (0, 1):
    for work in (0, 1500):
        for grid in (sms,) if work else (sms, 64, 32):
            for v in sorted(names):
                ctr = torch.zeros(64 * 32, dtype=torch.int32, device="cuda")
                flags = torch.zeros(256 * 32, dtype=torch.int32, device="cuda")
                ns = torch.zeros(256, dtype=torch.int64, device="cuda")
                cl.check(lib.dl_bench_grid_barrier(v, iters, traffic, work, ctr.data_ptr(), flags.data_ptr(), stream_buf.data_ptr(),
                                                   stream_buf.numel(), ns.data_ptr(), grid, cl.stream_ptr()), "bench_grid_barrier")
                torch.cuda.synchronize()
                t = ns[:grid].float().mean().item() / iters / 1e3
                print(f"traffic={traffic} stagger_ns={work:5d} grid={grid:3d} variant {v} [{names[v]}]: {t:6.3f} us/barrier", flush=True)
