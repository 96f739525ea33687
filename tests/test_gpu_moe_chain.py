"""Qwen3-MoE prompt prefill and decode steps through the engine (dl_engine_prefill, csrc/cuda/engine.cu) at production shapes,
chunk by chunk, against float64.

A MoE engine runs max_batch = 1: a prompt is tensor-core chunks of up to max_prefill tokens while at least tc_min_tokens remain
(enginePrefill, whose feed-forward is moePrefillFfn: router over the chunk -> sort by expert -> rmsnorm into pxn -> gather ->
grouped W1|W3 SwiGLU GEMM -> grouped W2 GEMM -> weighted combine), then one-token steps (engineForward(nb = 1): fused decode
attention, then runMoe: router -> expert-routed TMA GEMV with EPI_SWIGLU -> EPI_MOE_DOWN), which is also every decode step.

Stage checks (1-layer synthetic q40 models, attn_gain 2, a 4096-row context, from random bf16 or q80 K/V caches whose rows from
p0 + n on hold NaN): Qwen3-30B-A3B (dim 2048, 32 heads on 4 KV heads, 128 experts, 8 active, expert ff 768, 151936-token
vocabulary) and a Qwen3-235B-A22B geometry (dim 4096, 64 heads on 4 KV heads, 128 experts, 8 active, expert ff 1536, vocabulary
32002): kvMul 8 and 16. Every prompt runs one chunk per call with its plan asserted; after each chunk Engine.prefill_intermediates
and Engine.moe_intermediates give every stage's output, and each stage's float64 reference starts from the engine's own observed
input to that stage:
  * up to and including the WO residual: check_tc_attn / check_gemv_attn of test_gpu_prefill_chain.py, with its bounds.
  * router (test_gpu_moe.py): logits within 2^-18 |y| @ |gate|^T of the float64 rmsnorm y of the observed WO residual times the
    gate; ids exactly the top-k of the kernel's own logits, lowest index first on ties; weights within 2^-18 of the softmax of
    the chosen logits. Every later stage takes the kernel's routing.
  * tensor-core chunk: the MoE rmsnorm (bf16) bracketed around the float64 rmsnorm (2^-18 relative); each (token, slot) pair's h
    bracketed to bf16 around the float64 SwiGLU of that expert's tensor-core weights from the observed rmsnorm (2^-18 |a||w|
    accumulation, 2^-19 SiLU); the final residual within sum_j w_j 2^-18 |h_j| @ |W2_e|^T + 2^-22 of the magnitudes added, from
    the kernel's own bf16 h (prefill_check).
  * one-token step (decode_check): h per slot within the bound of the q80 activations of the float64 rmsnorm with their tie
    alternatives (q80_ref, 2^-18 relative input); the residual from the q80 of the kernel's own h per slot (2^-20 relative).
  * logits as in check_logits.
The WO residual x1 is overwritten by the combine: every chunk also runs with every expert's W2 block scales zeroed, whose final
residual is x1, and everything before W2 (scratch, routing and h) must be bitwise that of the normal run.

Negative controls perturb the float64 expectation and must miss their bound by 10x where they land furthest: token t's h combined
through token t + 1's experts and weights, one pair's expert replaced by the next expert id, gate and up rows swapped, routing weights left
unnormalised, plus the controls of check_tc_attn (attention without the diagonal and one row past it, the second chunk's K
rows rotated for p0 + t + 1, the WO residual of token t + 1) and the logits of token T - 2.

On an H100 80GB HBM3 (700 W power limit) the GPU tests of this file run in about 60 s, model writes included. Largest error /
bound over both shapes, both cache types and every prompt, from this file's Stats reports: tensor-core chunks QKV 0.77, q after
norm + RoPE 0.49, K rows 1.00 (q80 ints 0.998, scales 0.51), attention 0.52, WO residual 0.22, router logits 0.006, routing
weights 0.020, MoE residual 0.096, logits 0.013, and the MoE rmsnorm and every pair's h inside their bf16 brackets; one-token
steps QKV 0.007, q 0.009, attention 0.25, WO residual 0.017, router logits 0.005, routing weights 0.012, h per slot 0.001, MoE
residual 0.71 (q80 cache, 30B), logits 0.013. The stages up to WO use the dense chain's bounds and land near its figures there.
Weakest negative control over the shapes: attention without the diagonal 453x, one row past it 497x, gate and up rows swapped
4403x, K rows rotated one position 6120 ulps, token t's h combined through token t + 1's experts and weights 38937x, logits of
token T - 2 55773x, a pair routed to the next expert id 116287x, WO residual from token t + 1 149439x, routing weights
unnormalised 225699x.
No kernel source was mutated for this file.

Composition: the whole prompt in one call leaves the caches and logits bitwise equal to the chunk-by-chunk run, rows at p0 + n
and beyond stay NaN and no NaN reaches an output, and repeated runs are bitwise equal. The MoE scratch is process-wide and only
grows: a prompt gives bitwise equal caches and logits before and after a wider stand-alone call reallocates it (checked through
its capacities; this stands for a smaller model run after a larger one, whatever order the tests run in), and its read-back
refuses a shape other than the last call's. A 2-layer model decodes 16 greedy steps after a 391-token prompt with the decode
graph (which replays the router's and EPI_MOE_DOWN's self-resetting counters) and without it, bitwise equal. The engine's plan
is 192t 192t 1x7 for 391 tokens, never a GEMV batch wider than 1, and every token a one-token step when the expert ff is not a
multiple of 256 (planEnginePrefill's moeOk rule).

End to end (2 layers, 30B shape): the logits after a 391-token prompt and 16 greedy decode steps, and both layers' K/V rows,
against a float64 forward with bf16 activations on the tensor-core chunks and q80 ones on the one-token steps. Each layer takes
the experts its kernels chose: layer 1's are read back after every chunk and step, layer 0's from a 1-layer model written with
the same seed, whose layer-0 caches must be bitwise those of the 2-layer run. Measured tolerances E2E_*.
"""
import dataclasses
import gc
import time

import pytest
import torch

from q40_ref import (REL_NORM, Ref, Stats, _load, _random_caches, attention, bf16_ulp, f64_to_bf16, gemv, kv_rows, q80, q80_ref, ratio,
                     rms, rope_rows, silu, swiglu_ref)
from test_gpu_prefill_chain import (C_ACC, C_SUM, SEQ, TcWeights, _fmt, _poison_planes, _run_chunk, _same, _tokens, bf16_bracket_rel,
                                    bracket_ratio, c_acc, check_gemv_attn, check_logits, check_tc_attn, attn_ref, norm_rope, q_tc,
                                    tc_mm)

REL_H = 2.0 ** -20      # q80 of the kernel's own h: reciprocal and division only (test_gpu_moe.py)
TOL_W = 2.0 ** -18      # routing weights, absolute (test_gpu_moe.py)

NAMES = ["qwen3-30b-a3b", "qwen3-235b-a22b"]
MODEL_SEED = 53          # an n-layer model is written with seed MODEL_SEED + n
# (n, p0) per prompt: two tensor-core chunks then seven one-token steps; the shortest tensor-core chunk starting mid-tile; a chunk
# ending on the cache's last row; one-token steps only
PROMPTS = [(391, 0), (9, 37), (65, SEQ - 65), (7, 130)]


def _cfg(name, n_layers, **kw):
    from distributed_llama_b200.models.config import get_config
    cfg = get_config("qwen3-30b-a3b")
    if name == "qwen3-235b-a22b":
        cfg = dataclasses.replace(cfg, name=name, dim=4096, n_heads=64, n_kv_heads=4, head_dim=128, n_experts=128, n_active_experts=8,
                                  moe_hidden_dim=1536, vocab_size=32002)
    return dataclasses.replace(cfg, n_layers=n_layers, max_seq_len=SEQ, **kw)


class ExpertTc:
    """Tensor-core weights of a MoE Ref's experts (bf16, exact), built on first use."""

    def __init__(self, R):
        self.R, self.cache = R, {}

    def __call__(self, l, name, e):
        if (l, name, e) not in self.cache:
            self.cache[l, name, e] = self.R.expert_tc(l, name, e)
        return self.cache[l, name, e].double()


@pytest.fixture(scope="module")
def model(request, tmp_path_factory):
    """(name, n_layers) -> the synthetic model, its device weights and its float64 reference; one model at a time."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    name, n_layers = request.param
    cfg = _cfg(name, n_layers)
    path = str(tmp_path_factory.mktemp("moe_chain") / f"{name}-{n_layers}l.m")
    t0 = time.time()
    write_synthetic_model(path, cfg, seed=MODEL_SEED + n_layers, attn_gain=2.0)
    w = load_device_weights(ModelFile(path))
    R = Ref(path)
    assert R.n_experts == cfg.n_experts and R.ff == cfg.moe_hidden_dim
    print(f"\n[{name} x{n_layers}] model ready in {time.time() - t0:.1f} s")
    yield dict(name=name, cfg=cfg, weights=w, ref=R, tc=TcWeights(R), etc=ExpertTc(R))
    del w, R
    gc.collect()
    torch.cuda.empty_cache()


def _one(names):
    return pytest.mark.parametrize("model", [(n, 1) for n in names], indirect=True, ids=names)


def _engine(M, **kw):
    from distributed_llama_b200.runtime import Engine
    eng = Engine(M["weights"], **kw)
    assert eng.max_batch == 1 and not eng.mega
    return eng


# ------------------------------------------------------------------ MoE stage checks ------------------------------------------------------------------
def check_router(M, st, x1k, Mo, tag):
    """Router logits, ids and weights of rows x1k [T][dim] (f64, the observed WO residual) against float64."""
    R, L = M["ref"], M["ref"].layers[0]
    lg = Mo["logits"].view(x1k.shape[0], -1)
    y = rms(x1k, L["norm1"], R.eps)
    g = L["moe_gate"]
    st.r(f"{tag} router logits", ratio(lg, y @ g.T, C_ACC * (y.abs() @ g.abs().T)))
    want = torch.sort(lg, dim=1, descending=True, stable=True).indices[:, :R.k]
    assert torch.equal(Mo["ids"].view(-1, R.k).long(), want), f"{tag}: chosen experts differ from the top-k of the logits"
    sel = torch.gather(lg.double(), 1, want)
    wts = Mo["weights"].view(-1, R.k)
    st.r(f"{tag} routing weights", ratio(wts, torch.softmax(sel, 1), TOL_W))
    st.c("routing weights unnormalised", ratio(wts, torch.exp(sel - sel.amax(1, keepdim=True)), TOL_W))


def check_moe_tc(M, st, x1k, I, Mo, tag):
    """The MoE feed-forward of a tensor-core chunk: router, rmsnorm, h of every (token, slot) pair, final residual."""
    R, L, W = M["ref"], M["ref"].layers[0], M["etc"]
    T, k, ff = x1k.shape[0], R.k, R.ff
    check_router(M, st, x1k, Mo, tag)
    lo, hi = bf16_bracket_rel(rms(x1k, L["norm1"], R.eps), REL_NORM)
    st.r(f"{tag} moe rmsnorm (bracket)", bracket_ratio(I["xn"], lo, hi))
    xn, hk, ids, wts = I["xn"].double(), Mo["h"], Mo["ids"].long(), Mo["weights"].double()
    dx = torch.zeros(T, R.dim, dtype=torch.float64, device="cuda")
    tol, mag = torch.zeros_like(dx), torch.zeros_like(dx)
    for i, e in enumerate(ids.unique().tolist()):
        t, j = (ids == e).nonzero(as_tuple=True)
        a, got = xn[t], hk[t, j]
        w13 = W(0, "w13", e)
        gu = a @ w13.T
        eg = c_acc(w13) * (a.abs() @ w13.abs().T)
        h, eh = swiglu_ref(gu, eg)
        st.r(f"{tag} h per pair (bracket)", bracket_ratio(got, f64_to_bf16(h - eh), f64_to_bf16(h + eh)))
        if i < 4:
            hs, _ = swiglu_ref(gu.view(len(t), ff, 2).flip(-1).reshape(len(t), 2 * ff), eg)
            st.c("gate and up rows swapped", ratio(got, hs, eh + bf16_ulp(hs)))
            wn = W(0, "w13", (e + 1) % R.n_experts)
            hn, _ = swiglu_ref(a @ wn.T, eg)
            st.c("pair routed to the next expert id", ratio(got, hn, eh + bf16_ulp(hn)))
        w2 = W(0, "w2", e)
        hb = got.double()
        y = hb @ w2.T
        wt = wts[t, j][:, None]
        dx.index_add_(0, t, wt * y)
        tol.index_add_(0, t, wt * c_acc(w2) * (hb.abs() @ w2.abs().T))
        mag.index_add_(0, t, wt * y.abs())
    x2k = I["x"].double()
    b = tol + C_SUM * (mag + x2k.abs())
    st.r(f"{tag} moe residual", ratio(x2k, x1k + dx, b))
    if T >= 2:
        # token t's own h of slot j combined through token t + 1's expert and weight of slot j
        dn = torch.zeros(T - 1, R.dim, dtype=torch.float64, device="cuda")
        nxt = ids[1:]
        for e in nxt.unique().tolist():
            t, j = (nxt == e).nonzero(as_tuple=True)
            dn.index_add_(0, t, wts[t + 1, j][:, None] * (hk[t, j].double() @ W(0, "w2", e).T))
        st.c("token t combined with token t+1's routing", ratio(x2k[:-1], x1k[:-1] + dn, b[:-1]))


def check_moe_step(M, st, x1k, x2k, Mo, tag):
    """The MoE feed-forward of a one-token step: router, h per slot from the q80 rmsnorm, residual from the q80 of the kernel's h."""
    R, L = M["ref"], M["ref"].layers[0]
    check_router(M, st, x1k[None], Mo, tag)
    a1, amb1 = q80_ref(rms(x1k, L["norm1"], R.eps)[None], REL_NORM)
    dx = torch.zeros_like(x1k)
    tol, mag = torch.zeros_like(dx), torch.zeros_like(dx)
    for j, e in enumerate(Mo["ids"].tolist()):
        w13, s13 = R.expert_exact(0, "w13", e)
        gu = (a1 @ w13.T)[0]
        e_gu = (C_ACC * (a1.abs() @ s13.T) + amb1 @ w13.abs().T)[0]
        h, eh = swiglu_ref(gu, e_gu)
        st.r(f"{tag} h per slot", ratio(Mo["h"][j], h, eh))
        if j == 0:
            hs, _ = swiglu_ref(gu.view(R.ff, 2).flip(-1).reshape(-1), e_gu)
            st.c("gate and up rows swapped", ratio(Mo["h"][j], hs, eh))
            wn, _ = R.expert_exact(0, "w13", (e + 1) % R.n_experts)
            hn, _ = swiglu_ref((a1 @ wn.T)[0], e_gu)
            st.c("pair routed to the next expert id", ratio(Mo["h"][j], hn, eh))
        a2, amb2 = q80_ref(Mo["h"][j].double()[None], REL_H)
        w2, s2 = R.expert_exact(0, "w2", e)
        y = (a2 @ w2.T)[0]
        wt = float(Mo["weights"][j])
        dx += wt * y
        tol += wt * (C_ACC * (a2.abs() @ s2.T) + amb2 @ w2.abs().T)[0]
        mag += wt * y.abs()
    st.r(f"{tag} moe residual", ratio(x2k, x1k + dx, tol + C_SUM * (mag + x2k.abs())))


def run_prompt(M, eng, st, n, p0, caches, tag):
    """One prompt, one chunk per call (plan asserted), every stage checked after every chunk. Returns (caches, logits) after it."""
    toks = _tokens(n, p0, M["cfg"].vocab_size)
    plan = eng.prefill_plan(n, p0)
    assert all(tc or T == 1 for T, _, tc in plan), plan
    _load(eng, caches, poison_from=p0 + n)
    w2 = M["weights"].layers[0].w2
    saved = w2.scales.clone()
    n_tc = 0
    for T, p, tc in plan:
        part = toks[p - p0:p - p0 + T]
        w2.scales.zero_()
        try:
            _run_chunk(eng, part, p, (T, p, tc))
            I1, Mo1 = eng.prefill_intermediates(T, tc), eng.moe_intermediates(T, tc)
            x1k = (I1["x"] if tc else eng.x[:T]).double().clone()
        finally:
            w2.scales.copy_(saved)
        _run_chunk(eng, part, p, (T, p, tc))
        I, Mo = eng.prefill_intermediates(T, tc), eng.moe_intermediates(T, tc)
        logits = eng.logits[0].clone()
        for k in I:
            if tc and k == "h":
                continue          # the dense SwiGLU buffer, which a MoE chunk does not write (its h is Mo["h"])
            if k != "x":
                assert torch.equal(I1[k], I[k]), f"{tag} p={p}: {k} depends on W2's weights"
            assert not torch.isnan(I[k].float()).any(), f"{tag} p={p}: NaN in {k}"
        for k in Mo:
            assert torch.equal(Mo1[k], Mo[k]), f"{tag} p={p}: MoE {k} depends on W2's weights"
            assert not torch.isnan(Mo[k].float()).any(), f"{tag} p={p}: NaN in MoE {k}"
        assert torch.isfinite(logits).all(), f"{tag} p={p}: logits not finite"
        if tc:
            check_tc_attn(M, eng, st, part, p, I1, I, f"{tag} tc", second=n_tc == 1)
            check_moe_tc(M, st, x1k, I, Mo, f"{tag} tc")
            check_logits(M, st, logits, I["x"].double(), f"{tag} tc")
            n_tc += 1
        else:
            x2k = eng.x[:1].double()
            check_gemv_attn(M, eng, st, part[0], p, 1, I["qkv"][0], I["z"][0], x1k[0], f"{tag} step")
            check_moe_step(M, st, x1k[0], x2k[0], Mo, f"{tag} step")
            check_logits(M, st, logits, x2k, f"{tag} step")
    for c in _poison_planes(eng):
        assert torch.isnan(c[:, p0 + n:].float()).all(), f"{tag}: a row past the prompt was written"
        assert not torch.isnan(c[:, :p0 + n].float()).any(), f"{tag}: NaN in a row of the prompt or before it"
    if eng.kv_cache_float_type == "q80":
        for c, c0 in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
            assert torch.equal(c[:, p0 + n:], c0[:, p0 + n:]), f"{tag}: a q80 row past the prompt was written"


@pytest.mark.gpu
@_one(NAMES)
def test_moe_chain_against_float64(model):
    """Every stage of every chunk of the four prompts, and of a 256-token chunk (2048 pairs, the most moePrefillFfn takes), with
    bf16 and q80 caches, against float64 from the engine's own input to that stage; negative controls."""
    name = model["name"]
    st = Stats()
    t0 = time.time()
    for kv in ("bf16", "q80"):
        eng = _engine(model, kv_cache_float_type=kv)
        assert _fmt(eng.prefill_plan(391, 0)) == "192tx2 1x7"
        assert _fmt(eng.prefill_plan(9, 37)) == "9t" and _fmt(eng.prefill_plan(65, SEQ - 65)) == "65t"
        assert _fmt(eng.prefill_plan(7, 130)) == "1x7"
        caches = _random_caches(eng, 2026)
        for n, p0 in PROMPTS:
            run_prompt(model, eng, st, n, p0, caches, f"{name} {kv}")
        del eng
        eng = _engine(model, kv_cache_float_type=kv, max_prefill=256)
        assert _fmt(eng.prefill_plan(256, 0)) == "256t"
        run_prompt(model, eng, st, 256, 0, _random_caches(eng, 2027), f"{name} {kv} max_prefill 256")
        del eng
    print(f"\n[{name}] {time.time() - t0:.1f} s")
    st.report(name)


# ------------------------------------------------------------------ composition ------------------------------------------------------------------
def _fill(eng, caches, p0, n):
    _load(eng, caches, poison_from=p0 + n)
    eng.logits.fill_(float("nan"))


def _prompt_state(eng, toks, p0, caches, mode):
    """Caches and last logits after the prompt in one call ("whole") or one call per chunk ("chunks")."""
    n = len(toks)
    _fill(eng, caches, p0, n)
    if mode == "whole":
        eng.prefill(toks, p0)
    else:
        for T, p, tc in eng.prefill_plan(n, p0):
            _run_chunk(eng, toks[p - p0:p - p0 + T], p, (T, p, tc))
    torch.cuda.synchronize()
    logits = eng.logits[0].clone()
    assert torch.isfinite(logits).all(), f"n={n} p0={p0} {mode}: logits"
    for c in _poison_planes(eng):
        assert torch.isnan(c[:, p0 + n:].float()).all() and not torch.isnan(c[:, :p0 + n].float()).any(), f"n={n} p0={p0} {mode}"
    return [c.clone() for c in eng.k_cache + eng.v_cache + [s for s in eng.k_scale + eng.v_scale if s is not None]], logits


def _assert_same(a, b, what):
    for x, y in zip(a[0], b[0]):
        assert _same(x, y), f"{what}: caches differ"
    assert _same(a[1], b[1]), f"{what}: logits differ"


@pytest.mark.gpu
@_one(["qwen3-30b-a3b"])
@pytest.mark.parametrize("kv", ["bf16", "q80"])
def test_whole_prompt_equals_chunks(model, kv):
    """One dl_engine_prefill call over the whole prompt leaves the caches and the last logits bitwise those of one call per
    chunk; rows past the prompt (NaN) stay NaN and no NaN reaches an output; repeated runs are bitwise equal."""
    eng = _engine(model, kv_cache_float_type=kv)
    caches = _random_caches(eng, 11)
    for n, p0 in PROMPTS:
        toks = _tokens(n, p0, model["cfg"].vocab_size)
        ref = _prompt_state(eng, toks, p0, caches, "chunks")
        for mode in ("whole", "whole", "chunks"):
            _assert_same(ref, _prompt_state(eng, toks, p0, caches, mode), f"{kv} n={n} p0={p0} {mode}")


def _moe_scratch_caps():
    """Capacities of the process-wide MoE prefill scratch: pairs, dim, ff, experts, tokens."""
    import ctypes
    from distributed_llama_b200.ops import cuda_lib as cl
    out = (ctypes.c_uint64 * 5)()
    cl.lib().dl_moe_scratch_caps(out)
    return list(out)


def _grow_moe_scratch():
    """One stand-alone moePrefillFfn call one 256-column step wider than the scratch's dim capacity (ff 256, 128 experts, 256 tokens
    x 8 slots, one local expert, so its weights stay small). The scratch must be reallocated: its dim capacity is then that width."""
    from distributed_llama_b200.ops import DeviceQ40
    from distributed_llama_b200.ops import cuda_lib as cl
    before = _moe_scratch_caps()
    dim, ff, E, k, T = (before[1] + 511) // 256 * 256, 256, 128, 8, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    w13, w2 = DeviceQ40.empty(2 * ff, dim), DeviceQ40.empty(dim, ff)
    for w in (w13, w2):
        w.qs.copy_(torch.randint(-2 ** 31, 2 ** 31 - 1, w.qs.shape, generator=g, device="cuda", dtype=torch.int32))
        w.scales.copy_((torch.rand(w.scales.shape, generator=g, device="cuda") * 1e-3).half())
    x = torch.randn(T, dim, generator=g, device="cuda")
    norm = torch.ones(dim, device="cuda")
    gate = torch.randn(E, dim, generator=g, device="cuda") / dim ** 0.5
    xn = torch.empty(T, dim, dtype=torch.bfloat16, device="cuda")
    ids = torch.empty(T, k, dtype=torch.int32, device="cuda")
    wts = torch.empty(T, k, device="cuda")
    cl.check(cl.lib().dl_moe_prefill_ffn(x.data_ptr(), xn.data_ptr(), norm.data_ptr(), gate.data_ptr(), w13.qs.data_ptr(), w13.scales.data_ptr(),
                                         w2.qs.data_ptr(), w2.scales.data_ptr(), T, dim, ff, E, k, 0, 1, 1e-6,
                                         torch.cuda.get_device_properties(0).multi_processor_count, 0, ids.data_ptr(), wts.data_ptr(),
                                         cl.stream_ptr()), "moe_prefill_ffn")
    torch.cuda.synchronize()
    assert torch.isfinite(x).all()
    after = _moe_scratch_caps()
    assert after[1] == dim > before[1] and all(a >= b for a, b in zip(after, before)), (before, after)


@pytest.mark.gpu
@_one(["qwen3-30b-a3b"])
def test_moe_scratch_growth(model):
    """The MoE scratch is process-wide and its capacities only grow. A prompt (two 192-token chunks, one-token steps) gives bitwise
    equal caches and logits before and after a wider stand-alone call reallocates the scratch (asserted through its capacities;
    this stands for a smaller model run after a larger one in the same process, whatever order the tests run in), and so does a
    9-token chunk run after a 256-token one, whose rows past the chunk hold the earlier chunk's data. The scratch read-back refuses
    a chunk shape other than the last call's."""
    cfg = model["cfg"]
    eng = _engine(model)
    big = _engine(model, max_prefill=256)
    caches = _random_caches(eng, 17)
    toks = _tokens(391, 0, cfg.vocab_size)
    short = _tokens(9, 37, cfg.vocab_size)
    before = _prompt_state(eng, toks, 0, caches, "chunks")
    before_short = _prompt_state(eng, short, 37, caches, "chunks")
    _grow_moe_scratch()
    _assert_same(before, _prompt_state(eng, toks, 0, caches, "chunks"), "391 tokens after the scratch grew")
    _prompt_state(big, _tokens(256, 0, cfg.vocab_size), 0, caches, "chunks")
    _assert_same(before_short, _prompt_state(eng, short, 37, caches, "chunks"), "9 tokens after a 256-token chunk")
    assert eng.moe_intermediates(1, False)["ids"].shape == (8,)
    for rows in (8, 10):
        with pytest.raises(RuntimeError):
            eng.moe_intermediates(rows, True)
    assert eng.moe_intermediates(9, True)["ids"].shape == (9, 8)


@pytest.mark.gpu
def test_moe_engine_plans():
    """At the 30B geometry the plan is tensor-core chunks then one-token steps, never a GEMV batch wider than 1; with an expert ff
    of 384 (not a multiple of 256, so the grouped GEMMs cannot run) every token is a one-token step."""
    from distributed_llama_b200.models.loader import synthetic_device_weights
    from distributed_llama_b200.runtime import Engine
    for ff, tc in ((768, True), (384, False)):
        cfg = _cfg("qwen3-30b-a3b", 1, moe_hidden_dim=ff, vocab_size=32002)
        eng = Engine(synthetic_device_weights(cfg, max_seq_len=SEQ))
        assert eng.max_batch == 1
        for n, p0 in ((391, 0), (7, 130), (9, 37), (200, 100), (1, SEQ - 1), (65, SEQ - 65)):
            plan = eng.prefill_plan(n, p0)
            assert all(T == 1 or on for T, _, on in plan), plan
            assert sum(T for T, _, _ in plan) == n
            if not tc:
                assert plan == [(1, p0 + i, False) for i in range(n)], plan
        if tc:
            assert _fmt(eng.prefill_plan(391, 0)) == "192tx2 1x7"
            assert _fmt(eng.prefill_plan(200, 100)) == "192t 1x8"
        del eng
        gc.collect()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [("qwen3-30b-a3b", 2)], indirect=True, ids=["qwen3-30b-a3b"])
@pytest.mark.parametrize("kv", ["bf16", "q80"])
def test_decode_graph_equals_steps(model, kv):
    """2 layers: a 391-token prompt, then 16 greedy steps with the decode graph and without it give the same tokens, caches and
    final logits, bitwise; a second graph run repeats them."""
    cfg = model["cfg"]
    eng = _engine(model, kv_cache_float_type=kv)
    caches = _random_caches(eng, 23)
    toks = _tokens(391, 0, cfg.vocab_size)
    out = []
    for use_graph in (False, True, True):
        _fill(eng, caches, 0, 391 + 16)
        eng.prefill(toks, 0)
        first = int(eng.logits[0].argmax())
        gen = eng.decode_greedy(first, 391, 16, use_graph=use_graph)
        torch.cuda.synchronize()
        logits = eng.logits[0].clone()
        assert torch.isfinite(logits).all()
        for c in _poison_planes(eng):
            assert torch.isnan(c[:, 391 + 16:].float()).all() and not torch.isnan(c[:, :391 + 16].float()).any()
        out.append((gen, [c.clone() for c in eng.k_cache + eng.v_cache], logits))
    assert eng.graph_captured
    for gen, cs, lg in out[1:]:
        assert gen == out[0][0], f"{kv}: tokens differ with the decode graph"
        _assert_same((cs, lg), (out[0][1], out[0][2]), f"{kv}: decode graph")


# ------------------------------------------------------------------ end to end ------------------------------------------------------------------
# End to end, a bf16 or q80 rounding flip anywhere upstream moves later activations by a grid step, so these bounds are measured:
# on an H100 the largest errors were 0.0275 (logits, O(1) values), 0.0156 (first-layer K/V rows) and 0.0625 (second-layer K/V
# rows). The bounds leave a margin of 2x.
E2E_LOGITS = 0.055
E2E_KV = (0.03125, 0.125)
E2E_DECODE = 16


def forward_moe_ref(M, toks, plan, K, V, routes):
    """float64 forward of a prompt and its decode steps chunk by chunk (plan: (T, p, on tensor cores) from position 0): bf16
    activations on tensor-core chunks (attention over q~ as the tensor cores round it, h rounded to bf16), q80 on one-token steps.
    Every layer's MoE takes the experts its kernels chose (routes[l][chunk] [T][k]) with float64 softmax weights of float64 router
    logits. K, V: per layer f64 copies of the caches, updated in place with the bf16 rows. Returns the logits of the last token."""
    import math
    R, W, E = M["ref"], M["tc"], M["etc"]
    hd, nh, nkv, qd, kvd = R.hd, R.nh, R.nkv, R.q_dim, R.kv_dim
    logits = None
    for ci, (T, p, tc) in enumerate(plan):
        part = toks[p:p + T]
        if tc:
            x = torch.stack([R.embedding(t) for t in part])
            rows = R.rope[p:p + T]
            for l, L in enumerate(R.layers):
                qkv = tc_mm(W(l, "qkv"), f64_to_bf16(rms(x, L["norm0"], R.eps)))[0]
                q, _ = norm_rope(qkv[:, :qd].view(T, nh, hd), torch.zeros(T, nh, hd, dtype=torch.float64, device="cuda"), L["q_norm"],
                                 rows, R.eps)
                k = rms(qkv[:, qd:qd + kvd].view(T, nkv, hd), L["k_norm"], R.eps)
                K[l][:, p:p + T] = f64_to_bf16(rope_rows(k, rows)).transpose(0, 1)
                V[l][:, p:p + T] = f64_to_bf16(qkv[:, qd + kvd:].view(T, nkv, hd)).transpose(0, 1)
                z, _ = attn_ref(q_tc(q, hd), K[l], V[l], p, math.log(2))
                x = x + tc_mm(W(l, "wo"), f64_to_bf16(z.reshape(T, qd)))[0]
                y = rms(x, L["norm1"], R.eps)
                ids = routes[l][ci]
                wts = torch.softmax(torch.gather(y @ L["moe_gate"].T, 1, ids), 1)
                xn, dx = f64_to_bf16(y), torch.zeros_like(x)
                for e in ids.unique().tolist():
                    t, j = (ids == e).nonzero(as_tuple=True)
                    gu = xn[t] @ E(l, "w13", e).T
                    h = f64_to_bf16(silu(gu[:, 0::2]) * gu[:, 1::2])
                    dx.index_add_(0, t, wts[t, j][:, None] * (h @ E(l, "w2", e).T))
                x = x + dx
            logits = gemv(R.wcls, q80(rms(x[-1], R.final_norm, R.eps)), bound=False)[0]
        else:
            assert T == 1
            pos, x = p, R.embedding(part[0])
            for l, L in enumerate(R.layers):
                qkv, _ = gemv(L["qkv"], q80(rms(x, L["norm0"], R.eps)), bound=False)
                k, v = kv_rows(R, L, qkv, R.rope[pos])
                K[l][:, pos], V[l][:, pos] = f64_to_bf16(k), f64_to_bf16(v)
                z, _ = attention(qkv[:qd], K[l], V[l], pos + 1, L["q_norm"], R.rope[pos], nh, R.eps, 1, bound=False)
                x = x + gemv(L["wo"], q80(z), bound=False)[0]
                y = rms(x, L["norm1"], R.eps)
                ids = routes[l][ci][0]
                wts = torch.softmax(L["moe_gate"][ids] @ y, 0)
                act = q80(y)
                dx = torch.zeros_like(x)
                for j, e in enumerate(ids.tolist()):
                    gu, _ = gemv(L["w13"][e], act, bound=False)
                    dx += wts[j] * gemv(L["w2"][e], q80(silu(gu[0::2]) * gu[1::2]), bound=False)[0]
                x = x + dx
            logits = gemv(R.wcls, q80(rms(x, R.final_norm, R.eps)), bound=False)[0]
    return logits


def _run_routed(eng, toks, plan):
    """Runs the plan's chunks one call each; returns the last layer's expert ids per chunk and the last logits."""
    routes = []
    for T, p, tc in plan:
        if tc:
            _run_chunk(eng, toks[p:p + T], p, (T, p, tc))
        else:
            eng.step(toks[p], p)
            torch.cuda.synchronize()
        routes.append(eng.moe_intermediates(T, tc)["ids"].view(T, -1).long())
    return routes, eng.logits[0].clone()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [("qwen3-30b-a3b", 2)], indirect=True, ids=["qwen3-30b-a3b"])
def test_two_layers_end_to_end(model, tmp_path):
    """2 layers: a 391-token prompt and 16 greedy decode steps. The logits of the last step and both layers' K/V rows against the
    float64 forward with the routing each layer's kernels chose: layer 1's read back after every chunk and step, layer 0's from a
    1-layer model written with the same seed (the same embedding and layer 0), whose layer-0 caches must be bitwise those of the
    2-layer run."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    from distributed_llama_b200.runtime import Engine
    cfg = model["cfg"]
    n, steps = 391, E2E_DECODE
    eng = _engine(model)
    caches = _random_caches(eng, 99)
    prompt = _tokens(n, 0, cfg.vocab_size)
    _load(eng, caches)
    eng.prefill(prompt, 0)
    first = int(eng.logits[0].argmax())
    gen = eng.decode_greedy(first, n, steps)
    served = [c.clone() for c in eng.k_cache + eng.v_cache]
    toks = prompt + [first] + gen[:-1]
    plan = eng.prefill_plan(n, 0) + [(1, n + i, False) for i in range(steps)]
    assert _fmt(plan) == "192tx2 1x23"
    # the same inputs chunk by chunk, reading layer 1's routing; the caches must be those of the served run
    _load(eng, caches)
    routes1, got = _run_routed(eng, toks, plan)
    for a, b in zip(eng.k_cache + eng.v_cache, served):
        assert _same(a, b), "chunk-by-chunk caches differ from prefill + decode_greedy"
    # layer 0 alone
    path = str(tmp_path / "layer0.m")
    write_synthetic_model(path, _cfg(model["name"], 1), seed=MODEL_SEED + 2, attn_gain=2.0)
    eng0 = Engine(load_device_weights(ModelFile(path)))
    _load(eng0, ([caches[0][0]], [caches[1][0]]))
    routes0, _ = _run_routed(eng0, toks, plan)
    assert _same(eng0.k_cache[0], eng.k_cache[0]) and _same(eng0.v_cache[0], eng.v_cache[0]), "the 1-layer model's layer 0 differs"
    del eng0
    K = [c.double() for c in caches[0]]
    V = [c.double() for c in caches[1]]
    want = forward_moe_ref(model, toks, plan, K, V, [routes0, routes1])
    rows = n + steps
    err = {"logits": float((got.double() - want).abs().max())}
    for l in range(2):
        err[f"kv{l}"] = max(float((eng.k_cache[l][:, :rows].double() - K[l][:, :rows]).abs().max()),
                            float((eng.v_cache[l][:, :rows].double() - V[l][:, :rows]).abs().max()))
    print(f"\n[{model['name']} x2] max |error|: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    for k, v in err.items():
        lim = E2E_KV[int(k[2])] if k.startswith("kv") else E2E_LOGITS
        assert v <= lim, f"{k} off by {v:.3g} (bound {lim})"
