"""The persistent decode kernel (csrc/cuda/mega_decode.cu) at the per-layer shapes of production models, phase by phase against float64.

The kernel's GEMV geometry (row tiles, ring fills, segments per row, the step -> warp rotation) is derived on the host from the model
shape, and at test-model sizes most of it sits at a trivial value. Here every shape runs on synthetic 1- and 2-layer models with the
real dim / ffn / head geometry of Llama-3.1-8B, Llama-3.2-1B, Llama-3.2-3B, Qwen3-0.6B, Qwen3-14B and Llama-3.3-70B and a 4096-token
context.

Phase checks (1-layer models). Each phase's float64 reference starts from the kernel's own observed input to that phase
(`Engine.mega_vectors()`), so errors do not accumulate and every output element gets its own bound:
  * f32 accumulation: a small constant x 2^-24 x the sum of |terms| of that element;
  * q80 ties: an activation whose float64 rounding lies within the kernel's uncertainty of a tie (or a block whose fp16 scale does) is
    a discrete alternative. Where the phase's output is observed, the alternatives the kernel took are solved for (`gemv`) and
    only the accumulation bound remains; elsewhere each adds |W @ its change of xq|.
Negative controls perturb the float64 expectation and require the check to fail by at least 10x its bound: a row written with its
neighbour's value and a row that lost one 32-column block (each the median over the last row of every CTA's tile), attention over
one position too few or too many, and the K row rotated for the wrong position.

The W2 phase overwrites the WO residual x1 in place. To observe it, every position runs one extra launch with W2's block scales set to
zero: W2's row sums are then exactly 0 and the final residual is x1 itself. Nothing before W2 depends on W2's weights, so q|k|v, z
and the SwiGLU output of that launch must be bitwise those of the normal launch.
"""
import dataclasses
import gc
import time

import pytest
import torch

from q40_ref import U, Ref, attention, bf16_ulp, dequant, gemv, kv_rows, q80, rms, silu, worst

pytestmark = pytest.mark.gpu

SEQ = 4096
POSITIONS = [0, 1, 63, 64, 255, 256, 257, 1023, 1024, 2047, 2048, 4095]
CONTROL_MIN = 10.0               # a negative control must exceed its bound by this factor

# name: (preset, vocabulary of the synthetic model). Llama-3.1-8B keeps its real vocabulary (970/972-row logits tiles on 132 SMs);
# the others use an even vocabulary that leaves a pair remainder and a partial last ring fill in the logits phase.
SHAPES = {
    "llama-3.1-8b": ("llama-3.1-8b", 128256),
    "llama-3.2-1b": ("llama-3.2-1b", 32002),
    "llama-3.2-3b": ("llama-3.2-3b", 32002),
    "qwen3-0.6b": ("qwen3-0.6b", 32002),
    "qwen3-14b": ("qwen3-14b", 32002),
    "llama-3.3-70b": ("llama-3.3-70b", 32002),
}
NAMES = list(SHAPES)


def _cfg(preset, n_layers, vocab):
    from distributed_llama_b200.models.config import get_config
    return dataclasses.replace(get_config(preset), n_layers=n_layers, max_seq_len=SEQ, vocab_size=vocab)


def mega_geometry(cfg, grid):
    """launchMegaDecode's host geometry for a single-GPU model on `grid` CTAs, or None where the host code refuses the shape.

    A line-by-line replay of the host code in launchMegaDecode (csrc/cuda/mega_decode.cu): keep the two in step. It picks the rows
    the negative controls target (the last row of every CTA's tile) and the vocabularies that leave a partial logits fill. The
    engine exposes no geometry, so the tests check the replay where the kernel shows it: the phase tests assert that the
    persistent kernel ran for every shape it accepts, the grid test for every grid size it accepts."""
    hd = cfg.head_dim or cfg.dim // cfg.n_heads
    q_dim, kv_dim, ff = cfg.n_heads * hd, cfg.n_kv_heads * hd, cfg.hidden_dim
    ns = [cfg.dim, q_dim, ff, cfg.dim]
    if any(n % 128 for n in ns) or cfg.dim > 8192:
        return None
    max_n = max(ns)
    ds = [q_dim + 2 * kv_dim, cfg.dim, 2 * ff, cfg.dim, cfg.vocab_size]
    dn = [cfg.dim, q_dim, cfg.dim, ff, cfg.dim]
    partial = 16 * hd + 64
    for d, n in zip(ds, dn):
        if d % 2:
            return None
        partial = max(partial, (2 * ((d // 2 + grid - 1) // grid) + 2) * ((n // 32 + 31) // 32))
    partial = (partial + 3) // 4 * 4
    fixed = (max_n // 32) * 40 + partial * 4 + 32 * 4 + 2 * 128 * 4 + 2 * 16 * 8 + 256
    budget = 226 * 1024
    stage = max(36 * 1024, ((max_n // 32) * 18 * 4 + 127) // 128 * 128)
    if 2 * 64 * hd * 2 > stage or fixed + 2 * stage > budget:
        return None
    ph = []
    for d, n in zip(ds, dn):
        nseg = (n // 32 + 31) // 32
        sr = min(stage // ((n // 32) * 18) // 4 * 4, 64)
        g_inc = 16 // nseg
        ph.append(dict(d=d, n=n, nseg=nseg, stageRows=sr, pairsQ=d // 2 // grid, pairsRem=d // 2 % grid, gInc=g_inc,
                       segInc=16 - g_inc * nseg, rotInc=(sr // 4 * nseg) % 16))
    if 2 * (ph[1]["pairsQ"] + 1) > 512:
        return None
    return dict(stages=min((budget - fixed) // stage, 16), stageBytes=stage, ph=ph)


def tile(P, b):
    """(first row, rows) of CTA b's tile of a phase."""
    return 2 * (b * P["pairsQ"] + min(b, P["pairsRem"])), 2 * (P["pairsQ"] + (1 if b < P["pairsRem"] else 0))


# ------------------------------------------------------------------ float64 reference ------------------------------------------------------------------

def tile_ends(P, grid):
    """The last row of every CTA's tile of a phase."""
    return [sum(tile(P, b)) - 1 for b in range(grid) if tile(P, b)[1]]


def row_control(got, want, bound, rows):
    """Median over `rows` of error / bound when row r holds row r - 1's value."""
    r = torch.as_tensor(rows, device=want.device)
    return float(((got.double()[r] - want[r - 1]).abs() / bound[r]).median())


def lost_blocks(W, xq, rows):
    """Per row of `rows`: the contribution of its median-magnitude 32-column block (a lost segment of that row)."""
    r = torch.as_tensor(rows, device=W.device)
    c = (dequant(W[r])[0].double().view(len(rows), -1, 32) * xq.view(1, -1, 32)).sum(-1)
    return c.gather(1, c.abs().median(1, keepdim=True).indices)[:, 0], r


def block_control(got, want, bound, W, xq, rows):
    """Median over `rows` of error / bound when row r loses one 32-column block."""
    c, r = lost_blocks(W, xq, rows)
    return float(((got.double()[r] - (want[r] - c)).abs() / bound[r]).median())


def forward_ref(R, tok, p, K, V, n_splits):
    """float64 forward of one token at position p with q80 activations, per matrix (caches K, V: rows < p). Returns (logits, per layer
    (bf16 K row, bf16 V row))."""
    x = R.embedding(tok)
    rows = []
    rope_row = R.rope[p]
    for l, L in enumerate(R.layers):
        qkv, _ = gemv(L["qkv"], q80(rms(x, L["norm0"], R.eps)), bound=False)
        k, v = kv_rows(R, L, qkv, rope_row)
        kb, vb = k.to(torch.bfloat16), v.to(torch.bfloat16)
        rows.append((kb, vb))
        Kl, Vl = K[l].clone(), V[l].clone()
        Kl[:, p], Vl[:, p] = kb, vb
        z, _ = attention(qkv[:R.q_dim], Kl, Vl, p + 1, L["q_norm"], rope_row, R.nh, R.eps, n_splits, bound=False)
        x = x + gemv(L["wo"], q80(z), bound=False)[0]
        y, _ = gemv(L["w13"], q80(rms(x, L["norm1"], R.eps)), bound=False)
        hh = silu(y[0::2]) * y[1::2]
        x = x + gemv(L["w2"], q80(hh), bound=False)[0]
    logits, _ = gemv(R.wcls, q80(rms(x, R.final_norm, R.eps)), bound=False)
    return logits, rows


# ------------------------------------------------------------------ engines ------------------------------------------------------------------

def _engine(weights, monkeypatch, ctas=None, inflight=None):
    from distributed_llama_b200.runtime import Engine
    for var, val in (("DL_MEGA_CTAS", ctas), ("DL_MEGA_INFLIGHT", inflight)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    monkeypatch.delenv("DL_NO_MEGA", raising=False)
    monkeypatch.delenv("DL_MEGA_FLAGS", raising=False)   # bit 0 would select the experimental barrier-free hand-off
    eng = Engine(weights)            # enables the persistent kernel: the environment is read here
    return eng


def _random_caches(eng, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return ([torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.k_cache],
            [torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.v_cache])


def _load(eng, caches):
    for d, s in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
        d.copy_(s)


def _token(p, vocab):
    return (7919 * p + 11) % vocab


def _mega_step(eng, tok, p):
    eng.forward_batch([tok], p, logits_mode=1)
    torch.cuda.synchronize()
    assert eng.mega_active, "the step fell back to the multi-kernel path"
    eng.check_abort()


@pytest.fixture(scope="module")
def model(request, tmp_path_factory):
    """(name, n_layers) -> the synthetic model, its device weights and its float64 reference. One model at a time: the previous one is
    freed before the next is written."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    name, n_layers = request.param
    preset, vocab = SHAPES[name]
    cfg = _cfg(preset, n_layers, vocab)
    path = str(tmp_path_factory.mktemp("mega_shapes") / f"{name}-{n_layers}l.m")
    t0 = time.time()
    write_synthetic_model(path, cfg, seed=31 + n_layers, attn_gain=2.0)
    torch.cuda.reset_peak_memory_stats()
    w = load_device_weights(ModelFile(path))
    R = Ref(path)
    print(f"\n[{name} x{n_layers}] model ready in {time.time() - t0:.1f} s")
    yield dict(name=name, cfg=cfg, path=path, weights=w, ref=R)
    del w, R
    gc.collect()
    torch.cuda.synchronize()
    print(f"\n[{name} x{n_layers}] peak torch device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


def _one(names):
    return pytest.mark.parametrize("model", [(n, 1) for n in names], indirect=True, ids=names)


def _two(names):
    return pytest.mark.parametrize("model", [(n, 2) for n in names], indirect=True, ids=names)


# ------------------------------------------------------------------ tests ------------------------------------------------------------------

@_one(NAMES)
def test_phases_against_float64(model, monkeypatch):
    """Every phase of the persistent kernel at positions crossing the 64-row K/V chunk and 256-position split boundaries, against a
    float64 reference fed with the kernel's own input to that phase; write coverage (epochs, tails, poisoned outputs, only row p of
    the caches written); negative controls that prove each bound sees a row-level fault."""
    name, cfg, R = model["name"], model["cfg"], model["ref"]
    eng = _engine(model["weights"], monkeypatch)
    grid = eng.num_sms
    geo = mega_geometry(cfg, grid)
    assert geo is not None, f"{name}: the host geometry refuses the shape"
    P = geo["ph"][4]
    last_rows = [tile(P, b)[1] for b in range(eng.num_sms)]
    assert P["pairsRem"] > 0 and any(r % P["stageRows"] for r in last_rows), f"{name}: the vocabulary leaves no partial logits tile / fill"
    print(f"\n[{name}] stages {geo['stages']} x {geo['stageBytes']} B; " +
          "; ".join(f"{k}: nseg {p['nseg']} rows/fill {p['stageRows']} segInc {p['segInc']} rotInc {p['rotInc']} pairs {p['pairsQ']}+{p['pairsRem']}"
                    for k, p in zip(("qkv", "wo", "w13", "w2", "logits"), geo["ph"])))
    L = R.layers[0]
    K0, V0 = _random_caches(eng, 2024)
    ratios, controls = {}, {}

    def note(d, k, v):
        d[k] = max(d.get(k, 0.0), v) if d is ratios else min(d.get(k, float("inf")), v)

    w2 = model["weights"].layers[0].w2
    w2_scales = w2.scales.clone()
    prev_seq = None
    for p in POSITIONS:
        tok = _token(p, cfg.vocab_size)
        # the launch with W2 zeroed: its final residual is the kernel's x1
        _load(eng, (K0, V0))
        w2.scales.zero_()
        try:
            _mega_step(eng, tok, p)
        finally:
            w2.scales.copy_(w2_scales)
        vec1 = eng.mega_vectors()
        _load(eng, (K0, V0))
        eng.k_cache[0][:, p] = float("nan")
        eng.v_cache[0][:, p] = float("nan")
        eng.logits.fill_(float("nan"))
        _mega_step(eng, tok, p)
        vec = eng.mega_vectors()

        # ---- write coverage: one epoch per vector, a new launch sequence, zero tails, only row p of the caches ----
        seq = None
        for key, n, phase in (("x", R.dim, 5), ("qkv", R.q_dim + 2 * R.kv_dim, 1), ("z", R.q_dim, 2)):
            pay, ep = vec[key]
            e = int(ep[0])
            assert bool((ep[:n] == e).all()), f"{name} p={p}: {key} words carry several epochs"
            assert e & 1023 == phase, (key, e)
            seq = e >> 10 if seq is None else seq
            assert e >> 10 == seq
            assert bool((ep[n:] == 0).all()) and bool((pay[n:] == 0).all()), f"{name} p={p}: {key} tail words written"
        assert bool((vec["h"][R.ff:] == 0).all()), f"{name} p={p}: SwiGLU tail written"
        assert prev_seq is None or seq == prev_seq + 2          # the launch with W2 zeroed came in between
        prev_seq = seq
        assert int(vec1["x"][1][0]) >> 10 == seq - 1
        for key in ("qkv", "z"):
            assert torch.equal(vec1[key][0], vec[key][0]), f"{name} p={p}: {key} depends on W2's weights"
        assert torch.equal(vec1["h"], vec["h"]), f"{name} p={p}: the SwiGLU output depends on W2's weights"
        for got, src in ((eng.k_cache[0], K0[0]), (eng.v_cache[0], V0[0])):
            assert torch.equal(got[:, :p], src[:, :p]) and torch.equal(got[:, p + 1:], src[:, p + 1:]), f"{name} p={p}: a cache row other than p changed"
        logits = eng.logits[0].double()
        assert bool(torch.isfinite(logits).all()), f"{name} p={p}: logits not all written"

        qkv_k = vec["qkv"][0][:R.q_dim + 2 * R.kv_dim].double()
        z_k = vec["z"][0][:R.q_dim].double()
        h_k = vec["h"][:R.ff].double()
        x_k = vec["x"][0][:R.dim].double()
        x1_k = vec1["x"][0][:R.dim].double()
        rope_row = R.rope[p]

        # ---- 1. QKV: the input is the embedding row ----
        x0 = R.embedding(tok)
        xn = rms(x0, L["norm0"], R.eps)
        act = q80(xn, normed=True)
        xq = act[0]
        y, b = gemv(L["qkv"], act, got=qkv_k)
        note(ratios, "qkv", worst(qkv_k, y, b))
        ends = tile_ends(geo["ph"][0], grid)
        note(controls, "qkv row", row_control(qkv_k, y, b, ends))
        note(controls, "qkv block", block_control(qkv_k, y, b, L["qkv"], xq, ends))

        # ---- 2. the K/V row at p, from the kernel's raw k / v ----
        k, v = kv_rows(R, L, qkv_k, rope_row)
        got_k, got_v = eng.k_cache[0][:, p].double(), eng.v_cache[0][:, p]
        kb = k.to(torch.bfloat16).double()
        off = (got_k - kb).abs()
        assert bool((off <= bf16_ulp(kb)).all()), f"{name} p={p}: K row beyond 1 bf16 ulp ({float((off / bf16_ulp(kb)).max())})"
        n_off = int((off != 0).sum())
        assert n_off <= max(4, k.numel() // 64), f"{name} p={p}: {n_off} of {k.numel()} K elements are not the nearest bf16"
        note(ratios, "k ulp", float((off / bf16_ulp(kb)).max()))
        assert torch.equal(got_v, v.float().to(torch.bfloat16)), f"{name} p={p}: V row is not bf16(v)"
        pr = p + 1 if p + 1 < SEQ else p - 1
        kbad = kv_rows(R, L, qkv_k, R.rope[pr])[0].to(torch.bfloat16).double()
        note(controls, "rope p±1", float(((got_k - kbad).abs() / bf16_ulp(kbad)).max()))

        # ---- 3. attention: the kernel's q over the bf16 cache (its new row enters as bf16, like the cached ones) ----
        Kc, Vc = eng.k_cache[0], eng.v_cache[0]
        z, b = attention(qkv_k[:R.q_dim], Kc, Vc, p + 1, L["q_norm"], rope_row, R.nh, R.eps, eng.n_splits)
        note(ratios, "attention", worst(z_k, z, b))
        note(controls, "z row", row_control(z_k, z, b, [hh * R.hd + R.hd - 1 for hh in range(R.nh)]))
        for n_pos in (p, p + 2):
            if 1 <= n_pos <= SEQ:
                note(controls, "attention n±1", worst(z_k, attention(qkv_k[:R.q_dim], Kc, Vc, n_pos, L["q_norm"], rope_row, R.nh, R.eps,
                                                                     eng.n_splits, bound=False)[0], b))

        # ---- 4. WO + residual, from the kernel's attention output ----
        act = q80(z_k)
        zq = act[0]
        y_wo, b_wo = gemv(L["wo"], act, got=x1_k - x0)
        x1 = x0 + y_wo
        b_x1 = b_wo + U * x1.abs()
        note(ratios, "wo+residual", worst(x1_k, x1, b_x1))
        ends = tile_ends(geo["ph"][1], grid)
        note(controls, "x1 row", row_control(x1_k, x1, b_x1, ends))
        note(controls, "wo block", block_control(x1_k, x1, b_x1, L["wo"], zq, ends))

        # ---- 5. W1|W3 + SwiGLU, from the kernel's x1 ----
        act = q80(rms(x1_k, L["norm1"], R.eps), normed=True)
        xq = act[0]
        y13, b13 = gemv(L["w13"], act)
        g, u = y13[0::2], y13[1::2]
        sg = torch.sigmoid(g)
        hh = silu(g) * u
        b_h = (sg * (1 + g * (1 - sg))).abs() * u.abs() * b13[0::2] + silu(g).abs() * b13[1::2] + (16 + 2 * g.abs()) * U * hh.abs()
        note(ratios, "w13+swiglu", worst(h_k, hh, b_h))
        ends = [e // 2 for e in tile_ends(geo["ph"][2], grid)]      # the last SwiGLU output of every CTA
        note(controls, "h row", row_control(h_k, hh, b_h, ends))
        c, r = lost_blocks(L["w13"], xq, [2 * e for e in ends])  # its gate row loses a block
        note(controls, "w13 block", float(((h_k[r // 2] - silu(g[r // 2] - c) * u[r // 2]).abs() / b_h[r // 2]).median()))

        # ---- 6. W2 + residual, from the kernel's SwiGLU output and x1 ----
        act = q80(h_k)
        hq = act[0]
        y2, b2 = gemv(L["w2"], act, got=x_k - x1_k)
        x2 = x1_k + y2
        b_x = b2 + U * x2.abs()
        note(ratios, "w2+residual", worst(x_k, x2, b_x))
        ends = tile_ends(geo["ph"][3], grid)
        note(controls, "x row", row_control(x_k, x2, b_x, ends))
        note(controls, "w2 block", block_control(x_k, x2, b_x, L["w2"], hq, ends))

        # ---- 7. logits, from the kernel's final residual ----
        xn = rms(x_k, R.final_norm, R.eps)
        act = q80(xn, normed=True)
        xq = act[0]
        y, b = gemv(R.wcls, act, got=logits)
        note(ratios, "logits", worst(logits, y, b))
        ends = tile_ends(geo["ph"][4], grid)
        note(controls, "logits row", row_control(logits, y, b, ends))
        note(controls, "logits block", block_control(logits, y, b, R.wcls, xq, ends))

    print(f"\n[{name}] worst error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()))
    print(f"[{name}] weakest negative control / bound: " + ", ".join(f"{k} {v:.0f}" for k, v in controls.items()))
    for k, v in ratios.items():
        assert v <= 1.0, f"{name}: {k} exceeds its bound ({v:.3f})"
    for k, v in controls.items():
        assert v >= CONTROL_MIN, f"{name}: the negative control '{k}' is only {v:.1f}x its bound"


E2E_POSITIONS = [0, 64, 257, 2048, 4095]
# End to end, a q80 flip anywhere upstream moves later activations by one grid step, so these bounds are measured: on an H100 the
# largest errors over all shapes and positions were 0.052 (logits, O(1) values), 0.125 (second-layer K/V rows) and 0.0049
# (persistent vs multi-kernel logits). The bounds leave a margin of 2x, 2x and 4x. The first layer's K row is held to 1 bf16 ulp.
E2E_LOGITS = 0.1
E2E_KV = 0.25
E2E_PATHS = 0.02


@_two(NAMES)
def test_two_layers_end_to_end(model, monkeypatch):
    """2-layer models: logits and every layer's appended K/V row of the persistent kernel and of the multi-kernel path against the
    float64 per-matrix reference (q80 activations); the ring and the epochs carry on across the layer boundary."""
    name, cfg, R = model["name"], model["cfg"], model["ref"]
    eng = _engine(model["weights"], monkeypatch)
    caches = _random_caches(eng, 77)
    err = {}
    for p in E2E_POSITIONS:
        tok = _token(p, cfg.vocab_size)
        want, rows = forward_ref(R, tok, p, caches[0], caches[1], eng.n_splits)
        got = {}
        for path in ("mega", "multi"):
            eng.enable_mega(path == "mega")
            _load(eng, caches)
            eng.forward_batch([tok], p, logits_mode=1)
            torch.cuda.synchronize()
            assert eng.mega_active == (path == "mega")
            eng.check_abort()
            got[path] = eng.logits[0].double().clone()
            err[path] = max(err.get(path, 0.0), float((got[path] - want).abs().max()))
            for l, (kb, vb) in enumerate(rows):
                dk = float((eng.k_cache[l][:, p].double() - kb.double()).abs().max())
                dv = float((eng.v_cache[l][:, p].double() - vb.double()).abs().max())
                err[f"{path} kv{l}"] = max(err.get(f"{path} kv{l}", 0.0), dk, dv)
                if l == 0:
                    ulp = bf16_ulp(kb.double())
                    assert bool(((eng.k_cache[l][:, p].double() - kb.double()).abs() <= ulp).all()), f"{name} {path} p={p}: layer-0 K row"
        err["mega vs multi"] = max(err.get("mega vs multi", 0.0), float((got["mega"] - got["multi"]).abs().max()))
    print(f"\n[{name} x2] max |error|: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    for k, v in err.items():
        lim = E2E_KV if "kv" in k else E2E_PATHS if k == "mega vs multi" else E2E_LOGITS
        assert v <= lim, f"{name}: {k} off by {v:.3g} (bound {lim})"


VARIANTS = [(None, None), ("131", None), ("100", None), ("67", None), (None, "2"), (None, "0")]


@_one(["llama-3.1-8b", "qwen3-14b"])
def test_grid_and_pacing_invariance(model, monkeypatch):
    """The logits and every phase vector are bitwise equal across grid sizes (DL_MEGA_CTAS) and producer pacings (DL_MEGA_INFLIGHT):
    a row's arithmetic does not depend on which CTA owns it, which fill carries it or when the fill lands."""
    name, cfg = model["name"], model["cfg"]
    base = None
    for ctas, inflight in VARIANTS:
        eng = _engine(model["weights"], monkeypatch, ctas, inflight)
        if ctas is not None:
            assert mega_geometry(cfg, int(ctas)) is not None
        caches = _random_caches(eng, 5)
        out = []
        for p in (0, 257, SEQ - 1):
            _load(eng, caches)
            _mega_step(eng, _token(p, cfg.vocab_size), p)
            vec = eng.mega_vectors()
            out.append([eng.logits[0].clone(), vec["x"][0].clone(), vec["qkv"][0].clone(), vec["z"][0].clone(), vec["h"].clone(),
                        eng.k_cache[0][:, p].clone(), eng.v_cache[0][:, p].clone()])
        del eng
        if base is None:
            base = out
            continue
        for p, a, b in zip((0, 257, SEQ - 1), base, out):
            for what, x, y in zip(("logits", "x", "qkv", "z", "h", "k row", "v row"), a, b):
                assert torch.equal(x, y), f"{name} p={p}: {what} differs with DL_MEGA_CTAS={ctas} DL_MEGA_INFLIGHT={inflight}"


@_one(["llama-3.1-8b"])
def test_in_kernel_argmax(model, monkeypatch):
    """The arg-max at the end of the logits phase: tokens[0] = the first index of the maximum below the vocabulary limit, the position
    advances and history[p + 1] is written, eagerly and through the captured graph; ties between CTAs go to the lower index."""
    cfg, w = model["cfg"], model["weights"]
    V = cfg.vocab_size
    eng = _engine(w, monkeypatch)
    geo = mega_geometry(cfg, eng.num_sms)
    P = geo["ph"][4]
    b0, n0 = tile(P, 60)
    limits = [V, V - 1, b0 + n0 // 2 + 1, tile(P, 0)[1] - 3]
    caches = _random_caches(eng, 9)

    def check(limit, p, use_graph):
        _load(eng, caches)
        eng._set_inputs([_token(p, V)], p)
        eng.history.fill_(-1)
        eng.run_decode_step(use_graph=use_graph)
        torch.cuda.synchronize()
        assert eng.mega_active
        eng.check_abort()
        logits = eng.logits[0].cpu()
        want = int(torch.argmax(logits[:limit]))
        tok, pos = int(eng.tokens[0]), int(eng.pos[0])
        assert tok == want, f"limit {limit} p={p} graph={use_graph}: token {tok}, arg-max {want}"
        assert pos == p + 1 and int(eng.history[p + 1]) == tok
        return logits

    for limit in limits:
        eng.set_vocab_limit(limit)
        for p in (5, 1030):
            check(limit, p, False)
        check(limit, 300, True)

    # ties: the second half of the classifier duplicates the first, so every maximum has a twin in another CTA
    qs, sc = w.wcls.qs, w.wcls.scales
    saved = qs[V // 2:].clone(), sc[V // 2:].clone()
    qs[V // 2:] = qs[:V // 2]
    sc[V // 2:] = sc[:V // 2]
    try:
        eng = _engine(w, monkeypatch)
        for p, g in ((7, False), (2049, False), (400, True)):
            eng.set_vocab_limit(V)
            logits = check(V, p, g)
            assert torch.equal(logits[:V // 2], logits[V // 2:]), "duplicated rows do not give identical logits"
            a = int(eng.tokens[0])
            assert a < V // 2
            # a limit just above the maximum's twin: both twins stay admissible, every row after the twin is cut
            eng.set_vocab_limit(a + V // 2 + 1)
            check(a + V // 2 + 1, p, g)
            assert int(eng.tokens[0]) == a
    finally:
        qs[V // 2:], sc[V // 2:] = saved
