"""A/B of decode settings: runs `bench.py --gpus 1 --steps 64 --warmup 8` as subprocesses, alternating environment variants round by
round, checks that every run produced the same greedy tokens and prints median / min / max of the headline numbers per variant.

    python tools/ab_decode.py                                   # DL_MEGA_INFLIGHT=2 (the previous pacing) vs the default
    python tools/ab_decode.py --rounds 5 --variant DL_MEGA_INFLIGHT=2 --variant DL_MEGA_INFLIGHT=3 --variant ''
    python tools/ab_decode.py --variant 'DL_MEGA_INFLIGHT=2 DL_MEGA_CTAS=128' --variant ''
    python tools/ab_decode.py --variant @ab_checkouts/parent --variant ''      # another checkout of the code vs this tree

A variant is a space-separated list of NAME=VALUE settings; '' is the default environment. Every variant variable is removed from
the environment of the runs that do not set it. An item @DIR runs bench.py of the checkout at DIR (relative to this tree, e.g. a
`git archive` of another commit unpacked under the git-ignored ab_checkouts/) instead of this tree's; every checkout builds its
native libraries in place before the first round.
"""
import argparse
import io
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parse_variant(spec: str):
    """-> (environment settings, checkout root)"""
    env, root = {}, ROOT
    for item in spec.split():
        if item.startswith("@"):
            root = os.path.join(ROOT, item[1:])
            continue
        k, _, v = item.partition("=")
        env[k] = v
    return env, root


def gpu_info() -> str:
    exe = shutil.which("nvidia-smi")
    if not exe:
        return "nvidia-smi not found"
    r = subprocess.run([exe, "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True)
    return r.stdout.strip() or r.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--variant", action="append", default=None, help="NAME=VALUE ... ('' = default environment); repeatable")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--json", metavar="FILE", default=None, help="also write every run's result line to FILE")
    args = ap.parse_args()
    specs = args.variant if args.variant else ["DL_MEGA_INFLIGHT=2", ""]
    parsed = [parse_variant(s) for s in specs]
    variants = [env for env, _ in parsed]
    roots = [root for _, root in parsed]
    names = [s if s else "(default)" for s in specs]
    knobs = set().union(*variants)
    print(gpu_info(), flush=True)
    for root in dict.fromkeys(roots):
        r = subprocess.run([sys.executable, os.path.join(root, "__graft_entry__.py")], capture_output=True, text=True, cwd=root)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-3000:] + r.stderr[-3000:])
            raise SystemExit(f"build failed in {root}")

    results = {n: [] for n in names}
    tokens = []   # (variant, round, tokens.npy bytes)
    with tempfile.TemporaryDirectory() as tmp:
        for rnd in range(args.rounds):
            for name, var, root in zip(names, variants, roots):
                env = {k: v for k, v in os.environ.items() if k not in knobs}
                env.update(var)
                out = os.path.join(tmp, f"r{rnd}_{len(tokens)}")
                cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup",
                       str(args.warmup), "--dump-outputs", out]
                r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=root)
                lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                if r.returncode != 0 or not lines:
                    sys.stderr.write(r.stderr[-3000:])
                    raise SystemExit(f"bench.py failed for variant {name!r} (exit {r.returncode})")
                res = json.loads(lines[-1])
                results[name].append(res)
                with open(os.path.join(out, "tokens.npy"), "rb") as f:
                    tokens.append((name, rnd, f.read()))
                print(f"round {rnd} {name:40s} value {res['value']:8.2f}  pos2048 {res['extra'].get('decode_at_pos2048_tok_s')}"
                      f"  ttft {res['ttft_ms']:.3f} ms  sha {res['tokens_sha']}  agree {res['tokens_agree']}", flush=True)

    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)

    def stats(vals):
        return f"{statistics.median(vals):9.2f} {min(vals):9.2f} {max(vals):9.2f}"

    print(f"\n{'variant':40s} {'metric':24s} {'median':>9s} {'min':>9s} {'max':>9s}")
    for name in names:
        rs = results[name]
        print(f"{name:40s} {'value (tok/s)':24s} {stats([r['value'] for r in rs])}")
        print(f"{'':40s} {'decode_at_pos2048_tok_s':24s} {stats([r['extra']['decode_at_pos2048_tok_s'] for r in rs])}")
        print(f"{'':40s} {'ttft_ms':24s} {stats([r['ttft_ms'] for r in rs])}")
    if len(names) >= 2:
        base, new = names[0], names[-1]
        b = [r["value"] for r in results[base]]
        n = [r["value"] for r in results[new]]
        print(f"\n{new} vs {base}: median {statistics.median(n) / statistics.median(b) - 1:+.1%}, "
              f"slowest {new} {'>' if min(n) > max(b) else '<='} fastest {base}")

    ok = True
    shas = {r["tokens_sha"] for rs in results.values() for r in rs}
    if len(shas) != 1:
        print(f"MISMATCH: tokens_sha differs across runs: {sorted(shas)}")
        ok = False
    if not all(r["tokens_agree"] for rs in results.values() for r in rs):
        print("MISMATCH: tokens_agree is false in some run")
        ok = False
    ref = tokens[0][2]
    for name, rnd, blob in tokens:
        if blob != ref:
            print(f"MISMATCH: tokens.npy of {name} round {rnd} differs from the first run "
                  f"({np.load(io.BytesIO(blob))[:8]} vs {np.load(io.BytesIO(ref))[:8]})")
            ok = False
    print("tokens identical across all runs" if ok else "tokens DIFFER")
    raise SystemExit(0 if ok else 1)


if __name__ == "__main__":
    main()
