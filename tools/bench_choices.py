"""Throughput of n completions of one prompt: the batched choices step against n sequential single-sequence completions.

    python tools/bench_choices.py [--model llama-3.1-8b] [--tokens 64] [--repeats 3] [--controls]

On the synthetic q40 model of bench.py, one GPU, temperature 0.8 / top-p 0.9. For each prompt length and n it prefills the
prompt, then times the generation of `--tokens` tokens per choice (every choice runs to the limit: no stop token is checked)
with a host clock around work that ends in a device synchronise (every step reads its tokens back), after one untimed
warm-up run of the same shape. It prints one JSON line per measurement: aggregate generated tokens/s of the batched path and of
the sequential path (each choice in turn through the persistent single-token kernel), and the device time (CUDA events over
200 launches) of choiceAttnKernel alone at P = 2048 for B = 1 and 8 with the model's attention shape. The GPU name and
power limit are read in the same run. With --controls every measurement is also taken with the sampling controls on
(presence and frequency penalty 0.5, 100 logit_bias entries), alternating with the controls off (keys *_controls_tok_s).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Sequential:
    """The session with the batched path switched off: run_choices falls back to one choice after another."""

    def __init__(self, sess):
        self.sess = sess

    def batched_choices(self, n):
        return False

    def __getattr__(self, name):
        return getattr(self.sess, name)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_choices(sess, backend, prompt, n, tokens):
    import torch
    from distributed_llama_b200.api import run_choices
    sess.engine.prefill(prompt[:-1], 0, want_logits=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run_choices(backend, prompt[-1], len(prompt) - 1, n, tokens, sess.engine.seq_len, sess.sampler, 1234, lambda i, t: False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert all(len(o) == tokens for o in out)
    return sum(len(o) for o in out) / dt


CONTROLS = (0.5, 0.5, [(t, 1.0 if t % 2 else -1.0) for t in range(1000, 1100)])


def time_attention(eng, B, P, launches=200):
    import torch
    from distributed_llama_b200.ops import cuda_lib as cl
    w, h = eng.w, eng.w.header
    hd, n_heads, n_kv = h.head_dim, w.n_heads, w.n_kv_heads
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    seq = eng.seq_len
    C = (seq - 1 - P) // B
    qkv = torch.randn(B, q_dim + 2 * kv_dim, device="cuda")
    kc = (torch.randn(n_kv, seq, hd, device="cuda") * 0.1).bfloat16()
    vc = torch.randn(n_kv, seq, hd, device="cuda").bfloat16()
    partial = torch.empty(B * n_heads * eng.n_splits * (hd + 2), device="cuda")
    counters = torch.zeros(n_kv, dtype=torch.int32, device="cuda")
    out = torch.empty(B, q_dim, device="cuda")
    lib = cl.lib()

    def launch():
        cl.check(lib.dl_choice_attn_only(qkv.data_ptr(), q_dim + 2 * kv_dim, kc.data_ptr(), vc.data_ptr(), n_heads, n_kv, hd, seq,
                                         eng.n_splits, B, P, C, 0, 0, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim,
                                         cl.stream_ptr()), "dl_choice_attn_only")

    for _ in range(20):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama-3.1-8b")
    ap.add_argument("--tokens", type=int, default=64, help="generated tokens per choice")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--prompt-lens", default="64,2048")
    ap.add_argument("--ns", default="1,2,4,8")
    ap.add_argument("--controls", action="store_true", help="also time every measurement with sampling controls on")
    args = ap.parse_args()
    import torch
    from bench import ensure_model
    from distributed_llama_b200.api import InferenceSession
    assert torch.cuda.is_available(), "bench_choices needs a GPU"
    m, t = ensure_model(args.model)
    sess = InferenceSession(m, t, max_seq_len=4096, temperature=0.8, topp=0.9, seed=1234)
    gpu = gpu_info()
    for plen in map(int, args.prompt_lens.split(",")):
        prompt = [(7 * i + 3) % 1000 + 1 for i in range(plen)]
        for n in map(int, args.ns.split(",")):
            row = {"gpu": gpu, "prompt_len": plen, "n": n, "tokens_per_choice": args.tokens}
            variants = [("", (0.0, 0.0, []))] + ([("_controls", CONTROLS)] if args.controls else [])
            for name, backend in (("batched", sess), ("sequential", Sequential(sess))):
                if n == 1 and name == "sequential":
                    continue
                rates = {suffix: [] for suffix, _ in variants}
                for rep in range(args.repeats + 1):          # the first round is the warm-up
                    for suffix, ctl in variants:
                        sess.sampler.set_controls(*ctl)
                        r = time_choices(sess, backend, prompt, n, args.tokens)
                        if rep:
                            rates[suffix].append(r)
                for suffix, rs in rates.items():
                    rs.sort()
                    row[f"{name}{suffix}_tok_s"] = round(rs[len(rs) // 2], 1)
                    row[f"{name}{suffix}_tok_s_min_max"] = [round(rs[0], 1), round(rs[-1], 1)]
            print(json.dumps(row), flush=True)
    for B in (1, 8):
        us = time_attention(sess.engine, B, 2048)
        print(json.dumps({"gpu": gpu, "kernel": "choiceAttnKernel", "P": 2048, "B": B, "us": round(us, 2)}), flush=True)


if __name__ == "__main__":
    main()
