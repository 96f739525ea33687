"""Prompt prefill (dl_engine_prefill, csrc/cuda/engine.cu) at production shapes, chunk by chunk, against float64.

The engine splits a prompt into chunks (planPrefill): up to max_prefill tokens on the tensor cores (enginePrefill: rmsnorm -> QKV
GEMM -> QK-norm / RoPE / K/V append -> attention -> WO residual -> rmsnorm -> W1|W3 SwiGLU -> W2 residual) while at least
tc_min_tokens remain, then power-of-two GEMV batches (engineForward). The plan table pins that schedule without a GPU.

Stage checks (1-layer synthetic models with the dim / ffn / head geometry of Llama-3.1-8B with its 128256-token vocabulary,
Qwen3-14B, Qwen3-0.6B, Llama-3.2-1B and Llama-3.3-70B, and a 4096-token context, from random K/V caches). Every prompt runs one
chunk per call, each call's plan asserted, and after each chunk the engine's scratch (Engine.prefill_intermediates) gives every
stage's output. Each stage's float64 reference starts from the engine's own observed input to that stage:
  * tensor-core chunks: bf16 activations and weights rn_bf16(rn_bf16(f16 scale) * (q - 8)); f32 accumulation 2^-18 x sum |a w|
    (the bound of test_gpu_gemm_tc.py) up to K = 12288 columns and 2^-18 x K / 12288 x sum |a w| beyond, and 2^-22 of the
    magnitudes of split-K and residual sums. The tensor cores round once per k16 step, so the rounding error can grow with the
    K / 16 steps; with the SwiGLU outputs of a real chain as activations the Llama-3.3-70B W2 (K = 28672) reached 1.35 x 2^-18 in
    its worst element, and Qwen3-14B's (K = 17408) 0.88 x 2^-18, beyond the random-walk estimate that 2^-18 rests on. QKV, WO and
    W1|W3 (K <= 8192) keep 2^-18. Attention over q~ = bf16(q * log2(e) /
    sqrt(hd)) with (2^-9 + 2^-14) max|V| + 1 bf16 ulp (test_gpu_attn_prefill.py); bf16 stores bracketed. The first rmsnorm's
    output is overwritten before it can be read: it is bracketed to bf16, and an element whose bracket ends differ adds
    |W| x its bf16 step to the QKV bound. QK-norm carries the QKV bound through its derivative.
  * GEMV batches: q80 activations with their tie alternatives and the bounds of q40_ref.gemv / q40_ref.attention
    (test_gpu_mega_shapes.py).
  * K/V rows: bf16 within an ulp of the f64 QK-norm + RoPE of the kernel's raw k, V exactly bf16(v). With the q80 cache, the
    f16 scales and int8 values against a float64 q80 quantisation of the same rows, and attention over the cache as the kernels
    dequantise it (bf16-widened tiles on the tensor cores, exact on the CUDA cores); rows past the prompt carry NaN scales.
x1 (the WO residual) is overwritten by W2; every chunk also runs once with W2's block scales zeroed, whose final residual is x1,
and everything before W2 must be bitwise that of the normal run.

Negative controls perturb the float64 expectation and must exceed their bound 10x: the second chunk's K rows rotated for
p0 + t + 1, attention without the diagonal and with one row past it, the WO residual read from token t + 1 and the logits taken
from token T - 2. Row shifts count as the median over the chunk's tokens; a one-row attention shift is invisible to the late
tokens of a long random context, so the attention controls count where they land furthest.

On an H100 80GB HBM3 (700 W power limit) the GPU tests of this file run in about 90 s, model writes included. Largest error /
bound over all five shapes, every prompt and the variants: tensor-core chunks QKV 0.77, q after norm + RoPE 0.51 (QKV rows
rounded from a bracketed norm0), K rows 1.00 (ulp + RoPE rounding), attention 0.54, WO residual 0.31, W2 residual 0.62; GEMV
batches QKV 0.013, q 0.68, attention 0.23, WO 0.023, SwiGLU 0.89, W2 0.016; logits 0.017. The bf16 stores (post-attention
rmsnorm, SwiGLU) lie inside their rounding brackets. q80 cache: every scale is f16(amax / 127) exactly, the ints lie within
0.998 of their bound. Weakest negative control over the shapes: K rows rotated one position 7406 ulps, attention without the
diagonal 447x, one row past it 437x, WO residual from token t + 1 144377x, logits of token T - 2 27259x. No kernel source was
mutated for this file; the kernels' own mutation results are in the per-kernel tests.

Composition: the whole prompt in one call leaves the caches and the logits bitwise equal to the chunk-by-chunk run; rows at
p0 + n and beyond are NaN before the call and stay NaN, and no NaN reaches an output; slot prefill writes only its slot's rows,
with the values of the same chunks run without slots; repeated runs are bitwise equal.

End to end (2-layer models): logits and both layers' K/V rows of a 391-token prompt against a float64 forward with bf16
activations on the tensor-core chunks (attention over the bf16 q~ the tensor cores multiply) and q80 ones on the GEMV batches;
measured tolerances E2E_*.
"""
import dataclasses
import gc
import math
import time

import pytest
import torch

from q40_ref import (REL_NORM, U, Ref, Stats, _load, _random_caches, _scale_rows, attention, attn_operands, bf16_ulp,
                     check_kv_rows, f64_to_bf16, gemv, kv_rows, norm_rope, q40_parts, q80, ratio, rms, rope_rows, silu, swiglu_ref,
                     w_tc_of)

SEQ = 4096
C_ACC = 2.0 ** -18
K_ACC = 12288                      # the accumulation bound grows linearly with K beyond this many columns (see the docstring)
C_SUM = 2.0 ** -22
TOL_TC = 2.0 ** -9 + 2.0 ** -14
TOL_FALLBACK = 2e-4
LOG2E = 1.4426950408889634

SHAPES = {
    "llama-3.1-8b": ("llama-3.1-8b", 128256),
    "qwen3-14b": ("qwen3-14b", 32002),
    "qwen3-0.6b": ("qwen3-0.6b", 32002),
    "llama-3.2-1b": ("llama-3.2-1b", 32002),
    "llama-3.3-70b": ("llama-3.3-70b", 32002),
}
NAMES = list(SHAPES)
# (n, p0) per prompt: two tensor-core chunks then GEMV batches of 4, 2, 1; the shortest tensor-core chunk starting mid-tile; a
# chunk ending on the cache's last row; GEMV batches of 4, 2, 1
PROMPTS = [(391, 0), (9, 37), (65, SEQ - 65), (7, 130)]


# ------------------------------------------------------------------ plan table (no GPU) ------------------------------------------------------------------
def _plan(*a, **k):
    from distributed_llama_b200.runtime.engine import prefill_plan
    return prefill_plan(*a, **k)


PLAN_NS = [1, 7, 8, 9, 16, 191, 192, 193, 200, 201, 391]
# (minTc, maxPrefill, maxBatch, tensor cores allowed) -> chunk sizes per n in PLAN_NS ("t": on the tensor cores)
PLAN_TABLE = {
    (9, 192, 8, True): "1|4 2 1|8|9t|16t|191t|192t|192t 1|192t 8|192t 9t|192tx2 4 2 1",
    (9, 256, 8, True): "1|4 2 1|8|9t|16t|191t|192t|193t|200t|201t|256t 135t",
    (0, 192, 8, True): "1|4 2 1|8|8 1|8x2|8x23 4 2 1|8x24|8x24 1|8x25|8x25 1|8x48 4 2 1",
    (0, 256, 8, True): "1|4 2 1|8|8 1|8x2|8x23 4 2 1|8x24|8x24 1|8x25|8x25 1|8x48 4 2 1",
    (64, 192, 8, True): "1|4 2 1|8|8 1|8x2|191t|192t|192t 1|192t 8|192t 8 1|192tx2 4 2 1",
    (64, 256, 8, True): "1|4 2 1|8|8 1|8x2|191t|192t|193t|200t|201t|256t 135t",
    (9, 192, 1, True): "1|1x7|1x8|9t|16t|191t|192t|192t 1|192t 1x8|192t 9t|192tx2 1x7",
    (9, 256, 1, True): "1|1x7|1x8|9t|16t|191t|192t|193t|200t|201t|256t 135t",
    (0, 192, 1, True): "1|1x7|1x8|1x9|1x16|1x191|1x192|1x193|1x200|1x201|1x391",
    (0, 256, 1, True): "1|1x7|1x8|1x9|1x16|1x191|1x192|1x193|1x200|1x201|1x391",
    (64, 192, 1, True): "1|1x7|1x8|1x9|1x16|191t|192t|192t 1|192t 1x8|192t 1x9|192tx2 1x7",
    (64, 256, 1, True): "1|1x7|1x8|1x9|1x16|191t|192t|193t|200t|201t|256t 135t",
}
# without the tensor cores (dense f32 / f16 weights, MoE dims that are not multiples of 256) minTc and maxPrefill do not matter
PLAN_NO_TC = {8: "1|4 2 1|8|8 1|8x2|8x23 4 2 1|8x24|8x24 1|8x25|8x25 1|8x48 4 2 1",
              1: "1|1x7|1x8|1x9|1x16|1x191|1x192|1x193|1x200|1x201|1x391"}
# slot prefill: every chunk on the tensor cores, whatever its size and minTc
PLAN_SLOT = {192: "1t|7t|8t|9t|16t|191t|192t|192t 1t|192t 8t|192t 9t|192tx2 7t",
             256: "1t|7t|8t|9t|16t|191t|192t|193t|200t|201t|256t 135t"}


def _fmt(chunks):
    """'192t 192t 4 2 1', runs of equal sizes as '8x23'."""
    out = []
    for T, _, tc in chunks:
        s = f"{T}t" if tc else str(T)
        if out and out[-1][0] == s:
            out[-1][1] += 1
        else:
            out.append([s, 1])
    return " ".join(s if k == 1 else f"{s}x{k}" for s, k in out)


def _check_positions(chunks, n, p0):
    p = p0
    for T, q, _ in chunks:
        assert q == p, chunks
        p += T
    assert p == p0 + n, chunks


def test_plan_table():
    """The chunk lists of dl_prefill_plan for every n, p0, minTc, maxPrefill, maxBatch, tensor-core permission and slot prefill."""
    rows = SEQ
    for (min_tc, mp, mb, tc), want in PLAN_TABLE.items():
        for allowed in (True, False):
            row = want if allowed else PLAN_NO_TC[mb]
            for n, w in zip(PLAN_NS, row.split("|")):
                for p0 in (0, 37, rows - n):
                    got = _plan(n, p0, rows, mp, mb, min_tc, allowed)
                    _check_positions(got, n, p0)
                    assert _fmt(got) == w, f"n={n} p0={p0} minTc={min_tc} maxPrefill={mp} maxBatch={mb} tc={allowed}: {_fmt(got)}"
    slot_len = SEQ // 4
    for mp, want in PLAN_SLOT.items():
        for min_tc in (9, 0, 64):
            for allowed in (True, False):
                for n, w in zip(PLAN_NS, want.split("|")):
                    for p0 in (0, 37, slot_len - n):
                        got = _plan(n, p0, slot_len, mp, 8, min_tc, allowed, slot=1, slots=4)
                        _check_positions(got, n, p0)
                        assert _fmt(got) == w, f"slot n={n} p0={p0} maxPrefill={mp}: {_fmt(got)}"
    assert _plan(0, 5, rows, 192, 8, 9, True) == []


def test_plan_refusals():
    """A prompt past the cache (-60) and a slot prefill without slots (-64) are refused without a launch."""
    for n, p0 in ((1, SEQ), (2, SEQ - 1), (391, SEQ - 390), (SEQ + 1, 0)):
        with pytest.raises(RuntimeError, match="code -60"):
            _plan(n, p0, SEQ, 192, 8, 9, True)
    with pytest.raises(RuntimeError, match="code -60"):
        _plan(5, SEQ // 4 - 4, SEQ // 4, 192, 8, 9, True, slot=1, slots=4)
    for slots in (0, 1):
        with pytest.raises(RuntimeError, match="code -64"):
            _plan(5, 0, SEQ, 192, 8, 9, True, slot=0, slots=slots)
    assert _plan(1, SEQ - 1, SEQ, 192, 8, 9, True) == [(1, SEQ - 1, False)]


# ------------------------------------------------------------------ float64 pieces ------------------------------------------------------------------
class TcWeights:
    """The tensor-core weights of a Ref's matrices (rn_bf16(rn_bf16(f16 scale) * (q - 8)), exact in f32), built on first use."""

    def __init__(self, R):
        self.R, self.cache = R, {}

    def __call__(self, l, name):
        if (l, name) not in self.cache:
            raw = self.R.layers[l][name]
            d, nb = raw.shape[0], raw.shape[1]
            self.cache[l, name] = torch.cat([w_tc_of(*q40_parts(raw[r:r + 4096].reshape(-1, 18), min(4096, d - r), nb * 32)).float()
                                             for r in range(0, d, 4096)])
        return self.cache[l, name]


def c_acc(W):
    """f32 accumulation bound of a tensor-core GEMM over the columns of W, per unit of sum |a w|."""
    return C_ACC * max(1.0, W.shape[1] / K_ACC)


def tc_mm(W, a, extra=None):
    """float64 a @ W^T over rows [T][n] and S = |a| @ |W|^T (+ |extra| @ |W|^T: the bf16 step of bracketed inputs)."""
    ys, ss, es = [], [], []
    ad, aa = a.double(), a.double().abs()
    for r in range(0, W.shape[0], 8192):
        w = W[r:r + 8192].double()
        ys.append(ad @ w.T)
        w.abs_()
        ss.append(aa @ w.T)
        if extra is not None:
            es.append(extra @ w.T)
    return torch.cat(ys, 1), torch.cat(ss, 1), (torch.cat(es, 1) if extra is not None else 0)


def attn_ref(q, K, V, p0, c, shift=0):
    """softmax(c q . K^T) V of token t over positions 0 .. p0 + t + shift; q [T, H, hd], K, V [nkv, >= p0 + T, hd]. Returns
    f64 [T, H, hd] and max|V| over the visible rows [T, H]."""
    T, H, hd = q.shape
    nkv = K.shape[0]
    g = H // nkv
    P = p0 + T + max(shift, 0)
    qd = q.double().view(T, nkv, g, hd)
    hidden = torch.arange(P, device=q.device)[None, :] > (p0 + shift + torch.arange(T, device=q.device))[:, None]
    out = torch.empty(T, H, hd, dtype=torch.float64, device=q.device)
    for h in range(nkv):
        Kh, Vh = K[h, :P].double(), V[h, :P].double()
        s = torch.einsum("tgd,pd->tgp", qd[:, h], Kh) * c
        s.masked_fill_(hidden[:, None, :], float("-inf"))
        out[:, h * g:(h + 1) * g] = torch.einsum("tgp,pd->tgd", torch.softmax(s, -1), Vh)
    rowmax = V[:, :p0 + T].double().abs().amax(-1)
    vmax = torch.cummax(rowmax, 1).values[:, p0:].T.repeat_interleave(g, 1)
    return out, vmax


def q_tc(q, hd):
    """The bf16 q~ the tensor-core attention multiplies: bf16(f32(q) * f32(log2(e) / sqrt(hd)))."""
    s = torch.tensor(LOG2E, dtype=torch.float32) / torch.sqrt(torch.tensor(float(hd), dtype=torch.float32))
    return (q.float() * s.to(q.device)).bfloat16()


def bracket_ratio(got, lo, hi):
    """<= 1 iff every value lies in [lo, hi]: |got - mid| / half-width (an empty interval: 0 if equal)."""
    g = got.double()
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    d = (g - mid).abs()
    r = torch.where(half > 0, d / half.clamp_min(1e-300), torch.where(d == 0, torch.zeros_like(d), torch.full_like(d, float("inf"))))
    return float(torch.nan_to_num(r, nan=float("inf")).max())


def bf16_bracket_rel(r, rel):
    return f64_to_bf16(r - r.abs() * rel), f64_to_bf16(r + r.abs() * rel)


# ------------------------------------------------------------------ engines and models ------------------------------------------------------------------
def _cfg(preset, n_layers, vocab):
    from distributed_llama_b200.models.config import get_config
    return dataclasses.replace(get_config(preset), n_layers=n_layers, max_seq_len=SEQ, vocab_size=vocab)


@pytest.fixture(scope="module")
def model(request, tmp_path_factory):
    """(name, n_layers) -> the synthetic model, its device weights and its float64 reference; one model at a time."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    name, n_layers = request.param
    preset, vocab = SHAPES[name]
    cfg = _cfg(preset, n_layers, vocab)
    path = str(tmp_path_factory.mktemp("prefill_chain") / f"{name}-{n_layers}l.m")
    t0 = time.time()
    write_synthetic_model(path, cfg, seed=47 + n_layers, attn_gain=2.0)
    w = load_device_weights(ModelFile(path))
    R = Ref(path)
    print(f"\n[{name} x{n_layers}] model ready in {time.time() - t0:.1f} s")
    yield dict(name=name, cfg=cfg, weights=w, ref=R, tc=TcWeights(R))
    del w, R
    gc.collect()
    torch.cuda.empty_cache()


def _one(names):
    return pytest.mark.parametrize("model", [(n, 1) for n in names], indirect=True, ids=names)


def _two(names):
    return pytest.mark.parametrize("model", [(n, 2) for n in names], indirect=True, ids=names)


def _engine(weights, monkeypatch, no_tc_attn=False, **kw):
    from distributed_llama_b200.runtime import Engine
    if no_tc_attn:
        monkeypatch.setenv("DL_NO_TC_ATTN", "1")
    else:
        monkeypatch.delenv("DL_NO_TC_ATTN", raising=False)
    eng = Engine(weights, **kw)
    monkeypatch.delenv("DL_NO_TC_ATTN", raising=False)
    return eng


def _poison_planes(eng):
    """The planes that carry the NaN rows past a prompt: bf16 values, or q80 scales."""
    if eng.kv_cache_float_type == "q80":
        return [_scale_rows(eng, s) for s in eng.k_scale + eng.v_scale]
    return eng.k_cache + eng.v_cache


def _tokens(n, p0, vocab):
    return [(7919 * (p0 + i) + 11) % vocab for i in range(n)]


def _run_chunk(eng, toks, p, want):
    """One call that must run as exactly the chunk `want` = (T, p, on tensor cores)."""
    assert eng.prefill_plan(len(toks), p) == [want], (eng.prefill_plan(len(toks), p), want)
    eng.prefill(toks, p, want_logits=True)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ stage checks ------------------------------------------------------------------
def check_tc_chunk(M, eng, st, toks, p, I1, I, logits, tag, tc_attn=True, second=False):
    """Stage checks of a tensor-core chunk of T = len(toks) tokens at p from its scratch (I1: the run with W2 zeroed)."""
    R, L, W = M["ref"], M["ref"].layers[0], M["tc"]
    x1k = check_tc_attn(M, eng, st, toks, p, I1, I, tag, tc_attn, second)
    # post-attention rmsnorm, bracketed
    lo, hi = bf16_bracket_rel(rms(x1k, L["norm1"], R.eps), REL_NORM)
    st.r(f"{tag} rmsnorm1 (bracket)", bracket_ratio(I["xn"], lo, hi))
    # W1|W3 + SwiGLU, bracketed to bf16
    gu, S, _ = tc_mm(W(0, "w13"), I["xn"])
    h, e = swiglu_ref(gu, c_acc(W(0, "w13")) * S)
    lo, hi = f64_to_bf16(h - e), f64_to_bf16(h + e)
    st.r(f"{tag} w13+swiglu (bracket)", bracket_ratio(I["h"], lo, hi))
    # W2 residual
    x2k = I["x"].double()
    y, S, _ = tc_mm(W(0, "w2"), I["h"])
    x2 = x1k + y
    b = c_acc(W(0, "w2")) * S + C_SUM * (S + x1k.abs() + x2.abs())
    st.r(f"{tag} w2+residual", ratio(x2k, x2, b))
    check_logits(M, st, logits, x2k, tag)


def check_tc_attn(M, eng, st, toks, p, I1, I, tag, tc_attn=True, second=False):
    """The stages of a tensor-core chunk up to and including the WO residual: QKV, q after QK-norm and RoPE, the K/V rows,
    attention and WO. I1: the run whose final residual is the WO residual x1; returns x1 as float64."""
    R, L, W = M["ref"], M["ref"].layers[0], M["tc"]
    T, hd, nh, nkv, qd, kvd = len(toks), R.hd, R.nh, R.nkv, R.q_dim, R.kv_dim
    rows = R.rope[p:p + T]
    x0 = torch.stack([R.embedding(t) for t in toks])
    # QKV from the bracketed norm0 output
    r0 = rms(x0, L["norm0"], R.eps)
    lo, hi = bf16_bracket_rel(r0, REL_NORM)
    xn0 = f64_to_bf16(r0)
    y, S, E = tc_mm(W(0, "qkv"), xn0, extra=(hi - lo))
    b = c_acc(W(0, "qkv")) * S + E
    got = I["qkv"].double()
    st.r(f"{tag} qkv k|v", ratio(got[:, qd:], y[:, qd:], b[:, qd:]))
    q_ref, q_b = norm_rope(y[:, :qd].view(T, nh, hd), b[:, :qd].view(T, nh, hd), L["q_norm"], rows, R.eps)
    st.r(f"{tag} q (norm+rope)", ratio(got[:, :qd].view(T, nh, hd), q_ref, q_b))
    # K/V rows from the kernel's raw k, v
    k = got[:, qd:qd + kvd].view(T, nkv, hd)
    if L["k_norm"] is not None:
        k = rms(k, L["k_norm"], R.eps)
    kn, k = k, rope_rows(k, rows)
    check_kv_rows(eng, st, tag, p, k, kn, got[:, qd + kvd:].view(T, nkv, hd))
    Kc, Vc = attn_operands(eng, tc_attn)
    if second and eng.kv_cache_float_type == "bf16":
        kk = got[:, qd:qd + kvd].view(T, nkv, hd)
        if L["k_norm"] is not None:
            kk = rms(kk, L["k_norm"], R.eps)
        kbad = rope_rows(kk, R.rope[p + 1:p + T + 1]).to(torch.bfloat16).double()
        st.c("K rows rotated for p0+t+1 (ulp)", float(((Kc[:, p:p + T].transpose(0, 1).double() - kbad).abs() / bf16_ulp(kbad)).amax((1, 2)).median()))
    # attention from the kernel's rotated q over the cache as it stands
    q = I["qkv"][:, :qd].view(T, nh, hd)
    z = I["z"].view(T, nh, hd).double()
    if tc_attn:
        qt = q_tc(q, hd)
        z_ref, vmax = attn_ref(qt, Kc, Vc, p, math.log(2))
        zb = TOL_TC * vmax[..., None] + bf16_ulp(z_ref)
    else:
        z_ref, vmax = attn_ref(q, Kc, Vc, p, 1 / math.sqrt(hd))
        zb = TOL_FALLBACK * vmax[..., None] + bf16_ulp(z_ref)
    st.r(f"{tag} attention", ratio(z, z_ref, zb))
    if tc_attn and T >= 2:
        zd, _ = attn_ref(qt[1:], Kc, Vc, p + 1, math.log(2), shift=-1)
        st.c("attention without the diagonal", ratio(z[1:], zd, zb[1:]))
        zp, _ = attn_ref(qt[:T - 1], Kc, Vc, p, math.log(2), shift=1)
        st.c("attention one row past the diagonal", ratio(z[:T - 1], zp, zb[:T - 1]))
    # WO residual from the kernel's bf16 attention output
    x1k = I1["x"].double()
    y, S, _ = tc_mm(W(0, "wo"), I["z"])
    x1 = x0 + y
    b = c_acc(W(0, "wo")) * S + C_SUM * (S + x0.abs() + x1.abs())
    st.r(f"{tag} wo+residual", ratio(x1k, x1, b))
    if T >= 2:
        xbad = x0[1:] + y[:-1]
        st.c("WO residual from token t+1", float(((x1k[:-1] - xbad).abs() / b[:-1]).amax(1).median()))
    return x1k


def check_logits(M, st, logits, xk, tag):
    R = M["ref"]
    act = q80(rms(xk[-1], R.final_norm, R.eps), normed=True)
    y, b = gemv(R.wcls, act, got=logits)
    st.r(f"{tag} logits", ratio(logits, y, b))
    if xk.shape[0] >= 2:
        yb, _ = gemv(R.wcls, q80(rms(xk[-2], R.final_norm, R.eps), normed=True), bound=False)
        st.c("logits of token T-2", float(((logits.double() - yb).abs() / b).median()))


def check_gemv_batch(M, eng, st, toks, p, I, x1k, x2k, logits, tag):
    """Stage checks of a GEMV batch of nb = len(toks) tokens at p (q is rotated in place for nb >= 2, raw for nb = 1)."""
    R, L = M["ref"], M["ref"].layers[0]
    for i, tok in enumerate(toks):
        check_gemv_attn(M, eng, st, tok, p + i, len(toks), I["qkv"][i], I["z"][i], x1k[i], tag)
        y13, b13 = gemv(L["w13"], q80(rms(x1k[i], L["norm1"], R.eps), normed=True))
        g, u = y13[0::2], y13[1::2]
        sg = torch.sigmoid(g)
        hh = silu(g) * u
        b_h = (sg * (1 + g * (1 - sg))).abs() * u.abs() * b13[0::2] + silu(g).abs() * b13[1::2] + (16 + 2 * g.abs()) * U * hh.abs()
        st.r(f"{tag} w13+swiglu", ratio(I["h"][i], hh, b_h))
        y2, b2 = gemv(L["w2"], q80(I["h"][i].double()), got=x2k[i] - x1k[i])
        x2 = x1k[i] + y2
        st.r(f"{tag} w2+residual", ratio(x2k[i], x2, b2 + U * x2.abs()))
    check_logits(M, st, logits, x2k, tag)


def check_gemv_attn(M, eng, st, tok, pos, nb, qkv, zk, x1k, tag):
    """The stages of token `tok` at `pos` in a GEMV batch of nb up to and including the WO residual x1k (f64 [dim]): QKV, q
    (raw for nb = 1, after QK-norm and RoPE for nb >= 2), the K/V rows, attention and WO; qkv, zk: its rows of the scratch."""
    R, L = M["ref"], M["ref"].layers[0]
    hd, nh, qd, kvd = R.hd, R.nh, R.q_dim, R.kv_dim
    Kc, Vc = attn_operands(eng, False)
    ident = torch.stack([torch.ones(hd // 2), torch.zeros(hd // 2)], -1).double().cuda()
    x0 = R.embedding(tok)
    act = q80(rms(x0, L["norm0"], R.eps), normed=True)
    qkv = qkv.double()
    ykv, bkv = gemv(L["qkv"][qd:], act, got=qkv[qd:])
    st.r(f"{tag} qkv k|v", ratio(qkv[qd:], ykv, bkv))
    if nb == 1:
        yq, bq = gemv(L["qkv"][:qd], act, got=qkv[:qd])
        st.r(f"{tag} q", ratio(qkv[:qd], yq, bq))
    else:
        yq, bq = gemv(L["qkv"][:qd], act)
        q_ref, q_b = norm_rope(yq.view(1, nh, hd), bq.view(1, nh, hd), L["q_norm"], R.rope[pos:pos + 1], R.eps)
        st.r(f"{tag} q (norm+rope)", ratio(qkv[:qd].view(1, nh, hd), q_ref, q_b))
    k, v = kv_rows(R, L, qkv, R.rope[pos])
    kn = qkv[qd:qd + kvd].view(R.nkv, hd)
    check_kv_rows(eng, st, tag, pos, k[None], (kn if L["k_norm"] is None else rms(kn, L["k_norm"], R.eps))[None], v[None])
    zk = zk.double()
    if nb == 1:
        z, b = attention(qkv[:qd], Kc, Vc, pos + 1, L["q_norm"], R.rope[pos], nh, R.eps, eng.n_splits)
    else:
        z, b = attention(qkv[:qd], Kc, Vc, pos + 1, None, ident, nh, R.eps, eng.n_splits)
    st.r(f"{tag} attention", ratio(zk, z, b))
    y, b = gemv(L["wo"], q80(zk), got=x1k - x0)
    x1 = x0 + y
    st.r(f"{tag} wo+residual", ratio(x1k, x1, b + U * x1.abs()))


def run_prompt(M, eng, st, n, p0, caches, tag, tc_attn=True):
    """One prompt, one chunk per call (plan asserted), every stage checked after every chunk. Returns (caches, logits) after it."""
    cfg = M["cfg"]
    toks = _tokens(n, p0, cfg.vocab_size)
    plan = eng.prefill_plan(n, p0)
    _load(eng, caches, poison_from=p0 + n)
    w2 = M["weights"].layers[0].w2
    saved = w2.scales.clone()
    n_tc = 0
    for T, p, tc in plan:
        part = toks[p - p0:p - p0 + T]
        w2.scales.zero_()
        try:
            _run_chunk(eng, part, p, (T, p, tc))
            I1 = eng.prefill_intermediates(T, tc)
            x1k = eng.x[:T].double().clone()
        finally:
            w2.scales.copy_(saved)
        _run_chunk(eng, part, p, (T, p, tc))
        I = eng.prefill_intermediates(T, tc)
        logits = eng.logits[0].clone()
        for k in I:
            if k != "x":
                assert torch.equal(I1[k], I[k]), f"{tag} p={p}: {k} depends on W2's weights"
            assert not torch.isnan(I[k].float()).any(), f"{tag} p={p}: NaN in {k}"
        assert torch.isfinite(logits).all(), f"{tag} p={p}: logits not finite"
        if tc:
            check_tc_chunk(M, eng, st, part, p, I1, I, logits, f"{tag} tc", tc_attn=tc_attn, second=n_tc == 1)
            n_tc += 1
        else:
            check_gemv_batch(M, eng, st, part, p, I, x1k, eng.x[:T].double(), logits, f"{tag} gemv")
    for c in _poison_planes(eng):
        assert torch.isnan(c[:, p0 + n:].float()).all(), f"{tag}: a row past the prompt was written"
        assert not torch.isnan(c[:, :p0 + n].float()).any(), f"{tag}: NaN in a row of the prompt or before it"
    if eng.kv_cache_float_type == "q80":
        for c, c0 in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
            assert torch.equal(c[:, p0 + n:], c0[:, p0 + n:]), f"{tag}: a q80 row past the prompt was written"
    return [c.clone() for c in eng.k_cache], [c.clone() for c in eng.v_cache], eng.logits[0].clone()


@pytest.mark.gpu
@_one(NAMES)
def test_chain_against_float64(model, monkeypatch):
    """Every stage of every chunk of four prompts against float64 from the engine's own input to that stage; negative controls."""
    name = model["name"]
    eng = _engine(model["weights"], monkeypatch)
    eng.enable_mega(False)        # the last one-token batch runs the multi-kernel path, whose scratch the hook reads
    assert eng.prefill_plan(391, 0) == [(192, 0, True), (192, 192, True), (4, 384, False), (2, 388, False), (1, 390, False)]
    assert eng.prefill_plan(7, 130) == [(4, 130, False), (2, 134, False), (1, 136, False)]
    caches = _random_caches(eng, 2025)
    st = Stats()
    t0 = time.time()
    for n, p0 in PROMPTS:
        run_prompt(model, eng, st, n, p0, caches, name)
    print(f"\n[{name}] {time.time() - t0:.1f} s")
    st.report(name)


@pytest.mark.gpu
@_one(["llama-3.2-1b"])
def test_chain_variants(model, monkeypatch):
    """max_prefill = 256 with 257 tokens, tc_min_tokens = 0 with 20 tokens, the per-token attention inside enginePrefill
    (DL_NO_TC_ATTN=1) and the q80 KV cache (the four prompts), stage by stage."""
    w = model["weights"]
    st = Stats()
    eng = _engine(w, monkeypatch, max_prefill=256)
    eng.enable_mega(False)
    caches = _random_caches(eng, 7)
    assert eng.prefill_plan(257, 0) == [(256, 0, True), (1, 256, False)]
    run_prompt(model, eng, st, 257, 0, caches, "max_prefill 256")
    eng = _engine(w, monkeypatch)
    eng.enable_mega(False)
    eng.tc_min_tokens = 0
    assert eng.prefill_plan(20, 100) == [(8, 100, False), (8, 108, False), (4, 116, False)]
    run_prompt(model, eng, st, 20, 100, caches, "tc_min 0")
    eng = _engine(w, monkeypatch, no_tc_attn=True)
    eng.enable_mega(False)
    run_prompt(model, eng, st, 391, 0, caches, "no tc attn", tc_attn=False)
    eng = _engine(w, monkeypatch, kv_cache_float_type="q80")
    eng.enable_mega(False)
    q8 = _random_caches(eng, 8)
    for n, p0 in PROMPTS:
        run_prompt(model, eng, st, n, p0, q8, "q80 cache")
    st.report("variants")


# ------------------------------------------------------------------ composition ------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t.view(torch.int8) if t.dtype == torch.int8 else t.view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


@pytest.mark.gpu
@_one(["llama-3.1-8b", "qwen3-0.6b"])
@pytest.mark.parametrize("kv", ["bf16", "q80"])
def test_whole_prompt_equals_chunks(model, kv, monkeypatch):
    """One dl_engine_prefill call over the whole prompt leaves the caches and the last logits bitwise those of one call per
    chunk; rows past the prompt (NaN) stay NaN and no NaN reaches an output; repeated runs are bitwise equal."""
    w, cfg = model["weights"], model["cfg"]
    eng = _engine(w, monkeypatch, kv_cache_float_type=kv)
    g = torch.Generator(device="cuda").manual_seed(3)
    if kv == "bf16":
        caches = _random_caches(eng, 11)
    else:
        caches = ([torch.randint(-127, 128, c.shape, generator=g, device="cuda", dtype=torch.int8) for c in eng.k_cache],
                  [torch.randint(-127, 128, c.shape, generator=g, device="cuda", dtype=torch.int8) for c in eng.v_cache])
        scales = [(torch.rand(s.shape, generator=g, device="cuda") * 0.02 + 0.001).half() for s in eng.k_scale + eng.v_scale]
    for n, p0 in PROMPTS:
        toks = _tokens(n, p0, cfg.vocab_size)
        results = []
        for mode in ("chunks", "whole", "whole"):
            for d, s in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
                d.copy_(s)
                if kv == "bf16":
                    d[:, p0 + n:] = float("nan")
            if kv == "q80":
                for d, s in zip(eng.k_scale + eng.v_scale, scales):
                    d.copy_(s)
            eng.logits.fill_(float("nan"))
            if mode == "whole":
                eng.prefill(toks, p0)
            else:
                for T, p, tc in eng.prefill_plan(n, p0):
                    _run_chunk(eng, toks[p - p0:p - p0 + T], p, (T, p, tc))
            torch.cuda.synchronize()
            logits = eng.logits[0].clone()
            assert torch.isfinite(logits).all(), f"{kv} n={n} p0={p0} {mode}: logits"
            if kv == "bf16":
                for c in eng.k_cache + eng.v_cache:
                    assert torch.isnan(c[:, p0 + n:].float()).all() and not torch.isnan(c[:, :p0 + n].float()).any()
            results.append(([c.clone() for c in eng.k_cache + eng.v_cache], logits))
        for i in (1, 2):
            for a, b in zip(results[0][0], results[i][0]):
                assert _same(a, b), f"{kv} n={n} p0={p0}: caches differ between chunked and whole-prompt runs"
            assert _same(results[0][1], results[i][1]), f"{kv} n={n} p0={p0}: logits differ between chunked and whole-prompt runs"


@pytest.mark.gpu
@_one(["llama-3.1-8b"])
def test_slot_prefill(model, monkeypatch):
    """5- and 200-token prompts into slot 1 of 4 write only that slot's rows [0, n); every other row, NaN, is bitwise unchanged;
    the written rows equal those of the same tensor-core chunks run without slots. The engine refuses a slot prefill without
    slots and a prompt past the cache or the slot, in its plan and in dl_engine_prefill."""
    w, cfg = model["weights"], model["cfg"]
    for n in (5, 200):
        toks = _tokens(n, 0, cfg.vocab_size)
        ref = _engine(w, monkeypatch)
        ref.tc_min_tokens = 1
        plan = ref.prefill_plan(n, 0)
        for c in ref.k_cache + ref.v_cache:
            c.fill_(float("nan"))
        ref.prefill(toks, 0, want_logits=False)
        eng = _engine(w, monkeypatch)
        # the engine's refusals, before any launch: no slots yet (-64), a prompt past the cache (-60)
        with pytest.raises(RuntimeError, match="code -64"):
            eng.prefill_plan(n, 0, slot=1)
        with pytest.raises(RuntimeError, match="code -60"):
            eng.prefill_plan(n, SEQ - n + 1)
        with pytest.raises(RuntimeError, match="code -64"):
            eng._prefill(toks, 0, 1, False)
        with pytest.raises(RuntimeError, match="code -60"):
            eng._prefill(toks, SEQ - n + 1, -1, False)
        eng.set_slots(4)
        S = eng.slot_len
        with pytest.raises(RuntimeError, match="code -60"):
            eng.prefill_plan(n, S - n + 1, slot=1)
        assert eng.prefill_plan(n, 0, slot=1) == plan == [(min(n, 192), 0, True)] + ([(n - 192, 192, True)] if n > 192 else [])
        for c in eng.k_cache + eng.v_cache:
            c.fill_(float("nan"))
        before = [c.clone() for c in eng.k_cache + eng.v_cache]
        eng.slot_prefill(1, toks, 0)
        torch.cuda.synchronize()
        for c, c0, r in zip(eng.k_cache + eng.v_cache, before, ref.k_cache + ref.v_cache):
            blocks, blocks0 = c.view(4, c.shape[0], S, -1), c0.view(4, c.shape[0], S, -1)
            for s in (0, 2, 3):
                assert _same(blocks[s], blocks0[s]), f"n={n}: slot {s} changed"
            assert _same(blocks[1][:, n:], blocks0[1][:, n:]), f"n={n}: slot 1 rows past the prompt changed"
            assert _same(blocks[1][:, :n], r[:, :n]), f"n={n}: slot rows differ from the run without slots"
        del eng, ref


# ------------------------------------------------------------------ end to end ------------------------------------------------------------------
# End to end, a bf16 or q80 rounding flip anywhere upstream moves later activations by a grid step, so these bounds are measured:
# on an H100 the largest errors over all shapes were 0.020 (logits, O(1) values), 0.031 (first-layer K/V rows) and 0.125
# (second-layer K/V rows). The bounds leave a margin of 2x.
E2E_LOGITS = 0.04
E2E_KV = (0.0625, 0.25)


def forward_prompt_ref(M, toks, p0, plan, K, V):
    """float64 forward of the prompt chunk by chunk: bf16 activations on tensor-core chunks (attention over q~ as the tensor
    cores round it), q80 on GEMV batches. K, V: per
    layer f64 copies of the caches, updated in place with the bf16 rows. Returns the logits of the last token."""
    R, W = M["ref"], M["tc"]
    hd, nh, nkv, qd, kvd = R.hd, R.nh, R.nkv, R.q_dim, R.kv_dim
    logits = None
    for T, p, tc in plan:
        part = toks[p - p0:p - p0 + T]
        if tc:
            x = torch.stack([R.embedding(t) for t in part])
            rows = R.rope[p:p + T]
            for l, L in enumerate(R.layers):
                qkv = tc_mm(W(l, "qkv"), f64_to_bf16(rms(x, L["norm0"], R.eps)))[0]
                q, _ = norm_rope(qkv[:, :qd].view(T, nh, hd), torch.zeros(T, nh, hd, dtype=torch.float64, device="cuda"), L["q_norm"],
                                 rows, R.eps)
                k = qkv[:, qd:qd + kvd].view(T, nkv, hd)
                if L["k_norm"] is not None:
                    k = rms(k, L["k_norm"], R.eps)
                K[l][:, p:p + T] = f64_to_bf16(rope_rows(k, rows)).transpose(0, 1)
                V[l][:, p:p + T] = f64_to_bf16(qkv[:, qd + kvd:].view(T, nkv, hd)).transpose(0, 1)
                z, _ = attn_ref(q_tc(q, hd), K[l], V[l], p, math.log(2))
                x = x + tc_mm(W(l, "wo"), f64_to_bf16(z.reshape(T, qd)))[0]
                gu = tc_mm(W(l, "w13"), f64_to_bf16(rms(x, L["norm1"], R.eps)))[0]
                x = x + tc_mm(W(l, "w2"), f64_to_bf16(silu(gu[:, 0::2]) * gu[:, 1::2]))[0]
            logits = gemv(R.wcls, q80(rms(x[-1], R.final_norm, R.eps)), bound=False)[0]
        else:
            for i, tok in enumerate(part):
                pos = p + i
                x = R.embedding(tok)
                for l, L in enumerate(R.layers):
                    qkv, _ = gemv(L["qkv"], q80(rms(x, L["norm0"], R.eps)), bound=False)
                    k, v = kv_rows(R, L, qkv, R.rope[pos])
                    K[l][:, pos], V[l][:, pos] = f64_to_bf16(k), f64_to_bf16(v)
                    z, _ = attention(qkv[:qd], K[l], V[l], pos + 1, L["q_norm"], R.rope[pos], nh, R.eps, 1, bound=False)
                    x = x + gemv(L["wo"], q80(z), bound=False)[0]
                    y, _ = gemv(L["w13"], q80(rms(x, L["norm1"], R.eps)), bound=False)
                    x = x + gemv(L["w2"], q80(silu(y[0::2]) * y[1::2]), bound=False)[0]
                logits = gemv(R.wcls, q80(rms(x, R.final_norm, R.eps)), bound=False)[0]
    return logits


@pytest.mark.gpu
@_two(NAMES)
def test_two_layers_end_to_end(model, monkeypatch):
    """2-layer models, the 391-token prompt in one call (persistent kernel on for the last token, as served): logits and both
    layers' K/V rows against the float64 forward."""
    name, cfg = model["name"], model["cfg"]
    eng = _engine(model["weights"], monkeypatch)
    caches = _random_caches(eng, 99)
    n, p0 = 391, 0
    toks = _tokens(n, p0, cfg.vocab_size)
    _load(eng, caches)
    eng.prefill(toks, p0)
    torch.cuda.synchronize()
    got = eng.logits[0].double()
    K = [c.double() for c in caches[0]]
    V = [c.double() for c in caches[1]]
    want = forward_prompt_ref(model, toks, p0, eng.prefill_plan(n, p0), K, V)
    err = {"logits": float((got - want).abs().max())}
    for l in range(2):
        err[f"kv{l}"] = max(float((eng.k_cache[l][:, :n].double() - K[l][:, :n]).abs().max()),
                            float((eng.v_cache[l][:, :n].double() - V[l][:, :n]).abs().max()))
    print(f"\n[{name} x2] max |error|: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    for k, v in err.items():
        lim = E2E_KV[int(k[2])] if k.startswith("kv") else E2E_LOGITS
        assert v <= lim, f"{name}: {k} off by {v:.3g} (bound {lim})"
