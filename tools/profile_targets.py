"""Small driver for ncu captures: loads the 8B synthetic model, runs one prefill (tensor-core GEMM path) and a few decode steps."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import ensure_model
from distributed_llama_b200.api import InferenceSession

m, t = ensure_model("llama-3.1-8b")
sess = InferenceSession(m, t, max_seq_len=2048)
eng = sess.engine
prompt = [(7 * i + 3) % 1000 + 1 for i in range(128)]
eng.prefill(prompt[:-1], 0, want_logits=False)
out = eng.decode_greedy(prompt[-1], len(prompt) - 1, 6, use_graph=False)
torch.cuda.synchronize()
print("ok", out)
