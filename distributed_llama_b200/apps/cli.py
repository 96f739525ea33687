"""`dllama` command line: inference | chat | perplexity | worker (reference src/dllama.cpp:13-285)."""
from __future__ import annotations

import math
import os
import subprocess
import sys
import time
from typing import List

import numpy as np
import torch

from .. import host
from ..api import DraftRefused, draft_refusal
from .args import AppArgs, USAGE, parse_args
from .runtime import AppContext, run_inference_app, init_distributed_from_env


def _ms(dt: float) -> int:
    return int(dt * 1000)


def inference(ctx: AppContext) -> None:
    a = ctx.args
    if a.prompt is None:
        raise RuntimeError("Prompt is required")
    if a.steps == 0:
        raise RuntimeError("Number of steps is required")
    tok, inf, h = ctx.tokenizer, ctx.inference, ctx.header
    tokens = tok.encode(a.prompt, True, True)
    n_in = len(tokens)
    if n_in > h.seq_len:
        raise RuntimeError("The number of prompt tokens is greater than the sequence length")
    if n_in > a.steps:
        raise RuntimeError("The number of prompt tokens is greater than the number of steps")
    print(a.prompt)
    dev = ctx.sess.device
    eval_ms = 0.0
    pos = 0
    # prefill: all prompt tokens but the last (the reference evaluates nInputTokens-1 tokens in 32-token chunks; the
    # tensor-core path takes up to 256 tokens per chunk)
    chunk = 256 if inf.comm is None else a.n_batches
    while pos < n_in - 1:
        n = min(chunk, n_in - 1 - pos)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        inf.prefill(tokens[pos:pos + n], pos)
        torch.cuda.synchronize(dev)
        dt = (time.perf_counter() - t0) * 1000
        eval_ms += dt
        sent, recv = ctx.sess.engine.link_bytes(n)
        print(f"🔷️ Eval{int(dt):5d} ms Sync{0:5d} ms | Sent{sent // 1024:6d} kB Recv{recv // 1024:6d} kB | ({n} tokens)")
        pos += n
    sys.stdout.flush()
    token = tokens[pos]          # last prompt token (the reference reads one past it, SURVEY §7.3 — not copied)
    tok.reset_decoder()
    pred_ms = 0.0
    max_pos = min(h.seq_len, a.steps)
    greedy = ctx.sampler.temperature == 0.0
    ctx.sampler.begin_completion()
    n_pred = 0
    sync_prev = ctx.sess.engine.sync_ns() if inf.comm is not None else 0
    sync_total_us = 0
    spec = inf.speculates(ctx.sampler)
    while pos < max_pos:
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        # a speculative round emits several tokens: each line shows its share of the round's time
        toks = inf.spec_round(token, pos) if spec else [inf.next_token(token, pos, ctx.sampler)]
        dt = (time.perf_counter() - t0) * 1000
        pred_ms += dt
        for token in toks:
            piece = tok.decode(token).decode("utf-8", errors="replace")
            sent, recv = ctx.sess.engine.link_bytes(1)
            sync_now = ctx.sess.engine.sync_ns() if inf.comm is not None else 0
            sync_us, sync_prev = (sync_now - sync_prev) // 1000, sync_now
            sync_total_us += sync_us
            # Sync = time the decode kernel waited for peer ranks inside its fused all-reduces (a token takes ~1 ms: mostly prints 0;
            # the per-token average in microseconds is part of the summary)
            print(f"🔶 Pred{int(dt / len(toks)):5d} ms Sync{sync_us // 1000:5d} ms | Sent{sent // 1024:6d} kB Recv{recv // 1024:6d} kB | {piece if piece else '~'}")
            sys.stdout.flush()
            pos += 1
            n_pred += 1
            if pos >= max_pos:
                break
    n_eval = n_in - 1
    print()
    print("Evaluation")
    print(f"   nBatches: {chunk}")
    print(f"    nTokens: {n_eval}")
    if n_eval > 0 and eval_ms > 0:
        print(f"   tokens/s: {n_eval * 1000 / eval_ms:3.2f} ({eval_ms / n_eval:3.2f} ms/tok)")
    print("Prediction")
    print(f"    nTokens: {n_pred}")
    if n_pred > 0 and pred_ms > 0:
        print(f"   tokens/s: {n_pred * 1000 / pred_ms:3.2f} ({pred_ms / n_pred:3.2f} ms/tok)")
        if inf.comm is not None:
            print(f"   syncTime: {sync_total_us / n_pred:3.1f} us/tok (waiting for peer ranks inside the fused all-reduces)")
    if inf.draft is not None:
        print(inf.spec_stats.line())


def perplexity(ctx: AppContext) -> None:
    a = ctx.args
    if a.prompt is None:
        raise RuntimeError("Prompt is required")
    tok, inf, h = ctx.tokenizer, ctx.inference, ctx.header
    tokens = tok.encode(a.prompt, True, True)
    n = len(tokens)
    print(f"Evaluating {n} tokens...")
    total = 0.0
    for pos in range(n - 1):
        logits = inf.forward_logits(tokens[pos], pos).float()
        probs = torch.softmax(logits[: h.vocab_size], dim=-1)
        p = float(probs[tokens[pos + 1]])
        total += math.log(max(p, 1e-30))
        print(f"{pos + 1:5d} / {n - 1}, prob={p:f}")
    avg = total / max(1, n - 1)
    print()
    print("Results")
    print(f"   perplexity: {math.exp(-avg):f} (lower = better)")
    print(f"   avgLogProb: {avg:f}")
    print(f"   bitPerToken: {-avg / math.log(2.0):f}")


def make_chat_tools(ctx: AppContext):
    H = host()
    tok = ctx.tokenizer
    eos_ids = list(tok.eos_ids)
    stops = [tok.piece(i) for i in eos_ids]
    max_stop = max((len(s) for s in stops), default=0)
    ttype = H.parse_chat_template_type(ctx.args.chat_template) if ctx.args.chat_template else H.TEMPLATE_UNKNOWN
    gen = H.ChatTemplateGenerator(ttype, tok.chat_template, stops[0] if stops else b"")
    print(f"⭐ Chat template: {gen.type_name}")
    for s in stops:
        print(f"🛑 Stop: {s.decode('utf-8', errors='replace')}")
    det = H.EosDetector(eos_ids, stops, max_stop, max_stop)
    return gen, det


def chat(ctx: AppContext) -> None:
    H = host()
    tok, inf, h = ctx.tokenizer, ctx.inference, ctx.header
    gen, det = make_chat_tools(ctx)
    seq_len = h.seq_len
    sys_prompt = input("💻 System prompt (optional): ") if sys.stdin else ""
    items = []
    if sys_prompt:
        items.append(("system", sys_prompt))
    pos = 0
    greedy = ctx.sampler.temperature == 0.0
    while pos < seq_len:
        user = ""
        while not user:
            try:
                user = input("\n👱 User\n> ")
            except EOFError:
                return
        items.append(("user", user))
        content, public = gen.generate(items, True)
        tokens = tok.encode(content, pos == 0, True)
        end = min(seq_len, pos + len(tokens) - 1)
        n = end - pos
        inf.prefill(tokens[:n], pos)
        pos += n
        token = tokens[n] if n < len(tokens) else tokens[-1]
        tok.reset_decoder()
        det.reset()
        ctx.sampler.begin_completion()
        print("\n🤖 Assistant")
        if public:
            print(public.decode("utf-8", errors="replace"), end="")
        spec = inf.speculates(ctx.sampler)
        kind = None
        while pos < seq_len and kind != H.EOS:
            for token in (inf.spec_round(token, pos) if spec else [inf.next_token(token, pos, ctx.sampler)]):
                piece = tok.decode(token)
                kind = det.append(token, piece)
                if kind in (H.NOT_EOS, H.EOS):
                    delta = det.get_delta()
                    if delta:
                        print(delta.decode("utf-8", errors="replace"), end="", flush=True)
                    det.reset()
                pos += 1
                if kind == H.EOS or pos >= seq_len:
                    break
        items = []
    print("(end of context)")
    if inf.draft is not None:
        print(inf.spec_stats.line())


def worker(args: AppArgs) -> None:
    """`dllama worker`: in the one-process-per-GPU model a worker is simply a non-zero rank. It needs the same
    --model/--tokenizer flags as the root (every rank maps the model file and pulls only its own slices)."""
    comm = init_distributed_from_env()
    if comm is None or comm.rank == 0:
        raise RuntimeError("`dllama worker` must run as rank >= 1 of a torch.distributed job (use `dllama <mode> --gpus N`, "
                           "which spawns the root and its workers, or launch with torchrun)")
    run_inference_app(args, lambda ctx: None)


def _respawn_with_torchrun(argv: List[str], gpus: int) -> int:
    """`--gpus N`: start root + N-1 workers as N local processes (the GPU analogue of examples/n-workers.sh)."""
    port = 29500 + (os.getpid() % 2000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={gpus}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), "-m", "distributed_llama_b200.apps.cli"] + argv
    env = dict(os.environ, DLLAMA_SPAWNED="1")
    return subprocess.call(cmd, env=env)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    try:
        args = parse_args(argv, True)
        if args.help or args.mode is None:
            print(USAGE)
            return 0
        if args.draft_model is not None:
            why = draft_refusal(args.draft_tokens, max(args.gpus, 1, int(os.environ.get("WORLD_SIZE", "1"))) + len(args.workers))
            if why:
                raise DraftRefused(why)
        if args.gpus > 1 and os.environ.get("DLLAMA_SPAWNED") != "1" and int(os.environ.get("WORLD_SIZE", "1")) == 1:
            return _respawn_with_torchrun(argv, args.gpus)
        if args.mode == "inference":
            args.benchmark = True
            run_inference_app(args, inference)
        elif args.mode == "perplexity":
            run_inference_app(args, perplexity)
        elif args.mode == "chat":
            run_inference_app(args, chat)
        elif args.mode == "worker":
            worker(args)
        else:
            raise RuntimeError("Unsupported mode")
    except Exception as e:  # same contract as the reference: message + exit code 1
        print(f"🚨 Critical error: {e}")
        return 1
    finally:
        try:
            import torch.distributed as dist
            if dist.is_initialized():
                dist.destroy_process_group()
        except Exception:
            pass
    return 0


if __name__ == "__main__":
    sys.exit(main())
