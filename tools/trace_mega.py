"""Phase timeline of the persistent decode kernel (one %globaltimer stamp at every phase start on CTA 0).

    python tools/trace_mega.py [model] [--all] [--pos=N] [--kv=bf16|q80] [--save=FILE]

--pos=N traces the step at position N (default 63, the position after the 64-token prompt; the context is sized to fit it).
--kv=q80 runs with the q80 KV cache (--kv-cache-float-type), default bf16.
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from bench import ensure_model
from distributed_llama_b200.api import InferenceSession

args = [a for a in sys.argv[1:] if not a.startswith("--")]
ALL = "--all" in sys.argv          # every CTA records its stamps: barrier skew analysis
SAVE = next((a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--save=")), None)   # --all: also write the stamps (us) as .npy
POS = int(next((a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--pos=")), 63))
KV = next((a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--kv=")), "bf16")
model = args[0] if args else "llama-3.1-8b"
comm = None
rank = int(os.environ.get("RANK", "0"))
if int(os.environ.get("WORLD_SIZE", "1")) > 1:
    import torch.distributed as dist
    from distributed_llama_b200.parallel.comm import Communicator
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{os.environ['LOCAL_RANK']}"))
    comm = Communicator()
    if rank == 0:
        ensure_model(model)
    dist.barrier()
m, t = ensure_model(model)
sess = InferenceSession(m, t, max_seq_len=max(2048, POS + 64), comm=comm, kv_cache_float_type=KV)
eng = sess.engine
eng.enable_trace(4096, all_ctas=ALL)
eng.enable_mega()
prompt = [(7 * i + 3) % 1000 + 1 for i in range(64)]
eng.prefill(prompt[:-1], 0, want_logits=False)
eng.decode_greedy(prompt[-1], POS, 8)
torch.cuda.synchronize()
eng.trace_buf.zero_()
eng.decode_greedy(prompt[-1], POS, 1)
torch.cuda.synchronize()
if rank != 0:
    sys.exit(0)
L = eng.w.header.n_layers
if ALL:
    per_layer = ["qkv.pro", "qkv.main", "qkv.epi", "qkv.bar", "attn.run", "attn.bar", "wo.pro", "wo.main", "wo.epi", "wo.bar",
                 "w13.pro", "w13.main", "w13.epi", "w13.bar", "w2.pro", "w2.main", "w2.epi", "w2.bar"]
    names = ["embed"] + per_layer * L + ["logits.pro", "logits.main", "logits.epi"]
    nst = len(names) + 1
    T = eng.trace_buf.cpu().numpy().reshape(-1)[: eng.num_sms * eng.trace_stride].reshape(eng.num_sms, eng.trace_stride)[:, :nst].astype(np.float64)
    T = (T - T.min()) / 1e3          # us, common origin
    print(f"all-CTA trace at position {POS}: {eng.num_sms} CTAs x {nst} stamps; step = {T.max():.1f} us")
    # interval i spans stamps i..i+1; for a barrier interval the start stamp is the CTA's arrival and the end stamp its release
    stats = {}
    late = {}
    for i, nm in enumerate(names):
        a, r = T[:, i], T[:, i + 1]
        d = stats.setdefault(nm, {"dur": [], "skew": [], "lat": [], "wait": []})
        d["dur"].append(np.mean(r - a))
        if nm.endswith(".bar") or nm == "embed":
            last = a.max()
            d["skew"].append(last - a.min())
            d["wait"].append(np.mean(r - a))
            d["lat"].append(np.mean(r) - last)
            for c in np.argsort(-a)[:8]:
                late.setdefault(nm, {}).setdefault(int(c), 0)
                late[nm][int(c)] += 1
    print(f"{'interval':12s} {'mean dur':>9s} {'arrive skew':>12s} {'release-last':>13s}   (us, mean over layers; skew = last - first arrival)")
    for nm in ["embed"] + per_layer + ["logits.pro", "logits.main", "logits.epi"]:
        d = stats[nm]
        line = f"{nm:12s} {np.mean(d['dur']):9.2f}"
        if d["skew"]:
            line += f" {np.mean(d['skew']):12.2f} {np.mean(d['lat']):13.2f}"
        print(line)
    print("stragglers (CTA: times among the 8 latest arrivals, over the layers):")
    for nm, cnt in late.items():
        top = sorted(cnt.items(), key=lambda kv: -kv[1])[:10]
        print(f"  {nm:10s} " + " ".join(f"{c}:{n}" for c, n in top))
    # per-CTA main-loop durations: systematic fast/slow SMs?
    for ph in ("qkv.main", "wo.main", "w13.main", "w2.main"):
        idx = [i for i, nm in enumerate(names) if nm == ph]
        dur = np.stack([T[:, i + 1] - T[:, i] for i in idx], 1).mean(1)
        order = np.argsort(dur)
        print(f"  {ph}: per-CTA mean {dur.mean():.2f} us, min {dur.min():.2f} (cta {order[0]}), max {dur.max():.2f} (cta {order[-1]}), p90 {np.percentile(dur, 90):.2f}")
    # producer stalls (csrc/cuda/kernels.h megaTraceProdSlot): per weight phase k = 4 * layer + {QKV, WO, W1|W3, W2} (k = 4L: logits),
    # ns the producer waited for a free ring stage ("ring full") and on the in-flight cap; the qkv row includes the layer's K/V fills
    raw = eng.trace_buf.cpu().numpy().reshape(-1)[: eng.num_sms * eng.trace_stride].reshape(eng.num_sms, eng.trace_stride)
    p0 = (18 * L + 5 + 7) // 8 * 8
    P = raw[:, p0: p0 + 2 * (4 * L + 1)].astype(np.float64).reshape(eng.num_sms, 4 * L + 1, 2) / 1e3   # us
    full, cap = P[:, :, 0], P[:, :, 1]
    print(f"producer stalls (us per CTA, mean over {eng.num_sms} CTAs; per phase: mean over layers):")
    print(f"{'phase':8s} {'ring full':>10s} {'inflight cap':>13s}")
    for j, nm in enumerate(("qkv", "wo", "w13", "w2")):
        print(f"{nm:8s} {full[:, j:4 * L:4].mean():10.2f} {cap[:, j:4 * L:4].mean():13.2f}")
    print(f"{'logits':8s} {full[:, 4 * L].mean():10.2f} {cap[:, 4 * L].mean():13.2f}")
    fl = full[:, :4 * L].reshape(eng.num_sms, L, 4).sum(2).mean(0)
    cl_ = cap[:, :4 * L].reshape(eng.num_sms, L, 4).sum(2).mean(0)
    print(f"per layer total: ring full {fl.mean():.2f} us (min {fl.min():.2f}, max {fl.max():.2f}), "
          f"inflight cap {cl_.mean():.2f} us (min {cl_.min():.2f}, max {cl_.max():.2f})")
    print(f"per token: ring full {full.sum(1).mean():.1f} us, inflight cap {cap.sum(1).mean():.1f} us; step {T.max():.1f} us")
    if SAVE:
        np.save(SAVE, T)
    sys.exit(0)
st = eng.trace_buf.cpu().numpy().reshape(-1)
st = st[st != 0].astype(np.float64)
st = (st - st[0]) / 1e3
names = ["embed"]
for _ in range(L):
    names += ["qkv.pro", "qkv.main", "qkv.epi", "qkv.bar", "attn.run", "attn.bar", "wo.pro", "wo.main", "wo.epi", "wo.bar",
              "w13.pro", "w13.main", "w13.epi", "w13.bar", "w2.pro", "w2.main", "w2.epi", "w2.bar"]
names += ["logits.pro", "logits.main", "logits.epi"]
dur = np.diff(st)
print("total step us:", st[-1], "stamps", len(st), "expected", len(names) + 1)
agg = {}
for i, d in enumerate(dur):
    agg.setdefault(names[i] if i < len(names) else "?", []).append(d)
for nm, d in agg.items():
    print(f"{nm:12s} n={len(d):3d} mean={np.mean(d):7.2f} us  min={np.min(d):7.2f} max={np.max(d):7.2f}")
