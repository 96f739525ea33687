"""Greedy speculative decoding with a draft model (`--draft-model`) on synthetic q40 weights, one GPU.

    python tools/bench_speculative.py [--pairs llama-3.1-8b:llama-3.2-1b,qwen3-8b:qwen3-0.6b] [--tokens 128] [--repeats 3]

Per (target, draft) pair, with random-init weights in the device layout (models.loader.synthetic_device_weights):
* CUDA-event device times (median of 3 windows of 100 launches): one plain greedy step of the target and of the draft (persistent
  kernel, graph replay), and the target's verify forward (dl_engine_forward, logits mode 3) at nb = 2, 4 and 8;
* the host time of a whole round at k = 1, 3, 7 (graph replay, one result copy and synchronise), the break-even emitted tokens per
  round (round time / plain step time), and tokens/s and tokens per round over `--tokens` tokens after a 64-token prompt with
  - the draft equal to the target (a second engine on the target's weights: every draft accepted, the mechanism's upper bound),
  - the random draft of the pair (drafts almost never accepted: the overhead),
  against plain greedy decoding of the same tokens (decode_greedy, graph replay).
Synthetic weights say nothing about acceptance on real text; that stays unmeasured. One JSON line per pair with the GPU name and
power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def event_us(fn, windows=3, launches=100):
    import torch
    for _ in range(10):
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
    return round(sorted(ts)[len(ts) // 2], 1)


def median(xs):
    return sorted(xs)[len(xs) // 2]


def run_pair(target_name, draft_name, tokens, repeats, seq):
    import torch
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.loader import synthetic_device_weights
    from distributed_llama_b200.ops import cuda_lib as cl
    from distributed_llama_b200.runtime import Engine

    wt = synthetic_device_weights(get_config(target_name), seed=1, max_seq_len=seq)
    wd = synthetic_device_weights(get_config(draft_name), seed=2, max_seq_len=seq)
    tgt, same, drf = Engine(wt, seq_len=seq), Engine(wt, seq_len=seq), Engine(wd, seq_len=seq)
    prompt = [(7 * i + 3) % 1000 + 1 for i in range(64)]
    P = len(prompt) - 1
    for e in (tgt, same, drf):
        e.prefill(prompt[:-1], 0, want_logits=False)
    lib, sp = cl.lib(), cl.stream_ptr()
    out = {}

    # device times
    def step(e):
        return lambda: cl.check(lib.dl_engine_decode_graph(e._h, 1, sp), "decode_graph")
    for e in (tgt, drf):
        e._set_inputs([prompt[-1]], P)
    out["plain_step_us"] = event_us(step(tgt))
    out["draft_step_us"] = event_us(step(drf))
    tgt.verify(prompt[-8:], P)   # allocates the verify scratch
    verify = {}
    for nb in (2, 4, 8):
        tgt._set_inputs(prompt[-nb:], P)
        verify[nb] = event_us(lambda nb=nb: cl.check(lib.dl_engine_forward(tgt._h, nb, 3, 0, sp), "verify"))
    out["verify_us"] = verify

    def greedy():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        toks = tgt.decode_greedy(prompt[-1], P, tokens)
        return time.perf_counter() - t0, toks

    def spec(draft, k):
        tgt.prefill(prompt[:-1], 0, want_logits=False)
        draft.prefill(prompt[:-1], 0, want_logits=False)
        tok, pos, got, rounds, acc = prompt[-1], P, [], 0, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while len(got) < tokens:
            em, a, _ = tgt.spec_round(draft, tok, pos, k)
            got += em
            tok, pos, rounds, acc = em[-1], pos + len(em), rounds + 1, acc + a
        return time.perf_counter() - t0, got[:tokens], rounds, acc

    greedy()
    tg = []
    rows = {}
    for k in (1, 3, 7):
        for name, d in (("same", same), ("random", drf)):
            spec(d, k)   # the first round of each k runs eagerly and captures the round graph
    for _ in range(repeats):
        t, ref = greedy()
        tg.append(t)
        for k in (1, 3, 7):
            for name, d in (("same", same), ("random", drf)):
                t, got, rounds, acc = spec(d, k)
                r = rows.setdefault((k, name), {"t": [], "rounds": rounds, "accepted": acc, "equal": got == ref})
                r["t"].append(t)
    plain = tokens / median(tg)
    out["plain_tok_s"] = round(plain, 1)
    out["rounds"] = {}
    for k in (1, 3, 7):
        round_ms = {}
        for name in ("same", "random"):
            r = rows[(k, name)]
            t = median(r["t"])
            round_ms[name] = 1000 * t / r["rounds"]
            out["rounds"][f"k{k}_{name}"] = {"tok_s": round(tokens / t, 1), "speedup": round(tokens / t / plain, 3),
                                             "tokens_per_round": round(tokens / r["rounds"], 2),
                                             "acceptance": round(r["accepted"] / (k * r["rounds"]), 3),
                                             "round_ms": round(round_ms[name], 3), "tokens_equal_plain": r["equal"]}
        # break-even: a round pays when it emits more tokens than (round time / plain step time)
        out["rounds"][f"k{k}_break_even_tokens_per_round"] = round(round_ms["random"] * 1000 / out["plain_step_us"], 2)
    del tgt, same, drf, wt, wd
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="llama-3.1-8b:llama-3.2-1b,qwen3-8b:qwen3-0.6b")
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from tools.bench_parallel import gpu_info
    assert torch.cuda.is_available(), "bench_speculative needs a GPU"
    gpu = gpu_info()
    for pair in args.pairs.split(","):
        t, d = pair.split(":")
        res = run_pair(t, d, args.tokens, args.repeats, 1024)
        print(json.dumps({"gpu": gpu, "target": t, "draft": d, "tokens": args.tokens, **res}), flush=True)


if __name__ == "__main__":
    main()
