"""compute-sanitizer workload at the real Llama-3.1-8B shapes (random-init device weights): one tensor-core prefill chunk (GEMMs with
cooperative split-K, tensor-core attention, PDL chain) and three tokens of the persistent decode kernel.
    compute-sanitizer --tool memcheck python tools/sanitize_8b.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from distributed_llama_b200.models.config import get_config
from distributed_llama_b200.models.loader import synthetic_device_weights
from distributed_llama_b200.runtime import Engine
eng = Engine(synthetic_device_weights(get_config("llama-3.1-8b"), 0, 1, "cuda:0", max_seq_len=512))
eng.enable_mega()
prompt = [(7 * i + 3) % 1000 + 1 for i in range(40)]
eng.prefill(prompt[:-1], 0, want_logits=False)
toks = eng.decode_greedy(prompt[-1], len(prompt) - 1, 3, use_graph=False)
torch.cuda.synchronize()
print("llama-3.1-8b", "mega" if eng.mega_active else "multi-kernel", toks)
print("SANITIZE_TARGET_DONE")
