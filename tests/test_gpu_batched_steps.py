"""The batched decode steps, choices (dl_engine_choices_forward: n completions of one prompt, choiceAttnKernel) and slots
(dl_engine_slots_forward: --parallel N sequences in KV-cache slots, slotAttnKernel), at production shapes and long contexts
against float64, stage by stage.

The case table pins what each step runs without a GPU: the tile kernels' effective split count (ceil(nPos / 64), at most
n_splits), their query rows R (B * kvMul for choices, kvMul for slots) and dynamic shared memory (the mirror of TileSmem::bytes),
and the W2 GEMV plan of the batch. test_case_coverage asserts that the cases reach tile shared memory above 48 KB for both cache
types, one split, a split count that is not a power of two and the n_splits cap, a slot length that is not a multiple of 64, a
rotary position >= 65536 and the Llama-3.3-70B W2 batch of 8 that runs as two launches of 4.

Stage checks (1-layer synthetic q40 models with the attention and FFN geometry of Llama-3.1-8B (its 128256-token vocabulary,
131072 positions), Llama-3.2-1B, Llama-3.2-3B, Qwen3-14B (40960 positions), Qwen3-0.6B (its 151936-token vocabulary) and
Llama-3.3-70B; n_splits passed explicitly; bf16 and q80 caches filled with random rows). Every row the step must not read holds
NaN (bf16 values, or q80 scales): a choice's rows past j, an inactive choice's region, every row past the last choice, a slot's
rows past its position and an idle slot. Every step runs twice, the first time with W2's block scales zeroed, whose residual is
x1; everything before W2 must be bitwise that of the normal run. From the engine's own input to each stage:
  * QKV, WO + residual, W1|W3 + SwiGLU, W2 + residual and every row's logits: q80 activations with their tie alternatives and the
    bounds of q40_ref.gemv, batched over the rows of a step (q40_ref.gemv_rows); q after QK-norm and RoPE at the rotary position.
  * K/V rows at the cache row (choices: P + 1 + b * C + j, rotated for P + 1 + j; slots: row pos[b] of slot b): the bounds of
    check_kv_rows.
  * Attention over the exact row set (choices: [0, P] and [P + 1 + b * C, P + 1 + b * C + j]; slots: [0, pos[b]] of slot b), with
    the K/V operands as the tile kernels read them (bf16 as stored, q80 widened to f32 exactly) and a bound from the tile kernels'
    own order of operations (tile_attention).
Every cache row but the ones the step writes is bitwise unchanged (NaN rows stay NaN; inactive and padding rows write nothing), no
NaN reaches an active output, a changed token of an inactive row leaves the active rows' outputs bitwise unchanged, and at one
shape each slot's logits are bitwise those of the same step with every other slot idle. At Llama-3.2-3B the steps run twice in a
row (j, j + 1 and pos, pos + 1), so that the second step reads the row the first one stored.

Negative controls perturb the float64 expectation and must miss their bound 10x: the suffix K row rotated for its cache row, choice
b attending to choice b + 1's rows, slot b attending to slot b + 1's rows, attention without the step's new row and with one row
past it, row b's WO residual from row b + 1 and row b's logits from row b + 1's hidden state. Each counts where it lands furthest.

The kernel sweep runs dl_choice_attn_only and dl_slot_attn (bf16 and q80) alone at every (heads, kv heads, head dim) above, B 1, 3
and 8, either side of the split-count steps, against the same reference.

On an H100 80GB HBM3 (700 W power limit) the GPU tests of this file run in about 8 minutes, model writes included (Llama-3.1-8B
at 131072 positions about 160 s, every other shape 40-50 s, the kernel sweep under 10 s). Largest error / bound over all six shapes
and both cache types: choices QKV k|v 0.83, q after norm + RoPE 0.78, attention 0.088, WO residual 0.20, SwiGLU 0.90, W2 residual
0.015, logits 0.018; slots QKV k|v 0.60, q 0.38, attention 0.061, WO residual 0.12, SwiGLU 0.78, W2 residual 0.016, logits 0.88;
bf16 K rows 0.000 (every row the nearest bf16), q80 scales 0.000 and ints 0.998; kernel sweep: choice kernel 0.045, slot kernel
0.029. Weakest negative control over the shapes: logits of row b + 1 42410x, K row rotated for its cache row 288966 ulps, WO
residual from row b + 1 511126x, choice b attending to choice b + 1's rows 639196x, attention without the new row 4618950x; one
row past the new row and slot b attending to slot b + 1's rows land furthest on a one-row q80 output of exact zeros, whose bound
is the f32 underflow floor (about 1e37x there). No kernel source was mutated for this file.
"""
import dataclasses
import gc
import math
import time
import types

import pytest
import torch

from q40_ref import (U, Ref, Stats, _load, _random_caches, _scale_rows, bf16_ulp, check_kv_rows, gemv_rows, kv_rows, norm_rope, q80,
                     ratio, rms, rope, silu)

# name -> (preset, vocabulary, context, n_splits); n_splits are the engine's defaults on a 132-SM H100: 2 * 132 // heads
SHAPES = {
    "llama-3.1-8b": ("llama-3.1-8b", 128256, 131072, 8),
    "llama-3.2-1b": ("llama-3.2-1b", 32002, 32768, 8),
    "llama-3.2-3b": ("llama-3.2-3b", 32002, 32768, 11),
    "qwen3-14b": ("qwen3-14b", 32002, 40960, 6),
    "qwen3-0.6b": ("qwen3-0.6b", 151936, 32768, 16),
    "llama-3.3-70b": ("llama-3.3-70b", 32002, 32768, 4),
}
NAMES = list(SHAPES)
CONSECUTIVE = "llama-3.2-3b"     # the steps of its cases run twice in a row
ALONE = "qwen3-14b"              # each slot's logits against the same step with every other slot idle
C_OWN = 40                       # rows per choice: j = C - 1 ends a full tile and a partial one
KTILE = 32
SMEM_DEFAULT = 48 * 1024
SMEM_MAX = 227 * 1024
PLAIN, RESID = 1, 1              # the W2 GEMV: plain prologue, residual epilogue


# ------------------------------------------------------------------ case table (no GPU) ------------------------------------------------------------------
def geometry(name):
    from distributed_llama_b200.models.config import get_config
    c = get_config(SHAPES[name][0])
    hd = c.head_dim or c.dim // c.n_heads
    return c.n_heads, c.n_kv_heads, hd, c.dim, c.hidden_dim


def eff_splits(n_pos, n_splits):
    """effectiveSplit: ceil(nPos / 64) splits, at most n_splits."""
    return max(1, min(n_splits, -(-n_pos // 64)))


def tile_smem(hd, q8, R):
    """TileSmem<HD, Q8>::bytes(R): q and acc [R][HD] f32, m and l [R], one K and one V tile of 32 padded rows (f32 for q80)."""
    pad = hd + 1 if q8 else hd + 2
    return R * hd * 8 + R * 8 + 2 * KTILE * pad * (4 if q8 else 2)


def pow2(n):
    nb = 1
    while nb < n:
        nb *= 2
    return nb


def choice_runs(name):
    """(B, P, js, inactive choices, effective splits) per run: the steps j of js run in a row on one cache."""
    seq, ns = SHAPES[name][2:]
    C, cap = C_OWN, 64 * ns + 37
    runs = [(1, 0, (0,), (), 1), (3, 63, (C - 1,), (), 1), (8, 64, (C - 1,), (2,), 2), (8, cap, (0,), (), ns),
            (3, seq - 1 - 3 * C, (C - 1,), (), ns)]
    if name == CONSECUTIVE:
        runs.append((3, 64, (5, 6), (1,), 2))
    return runs


def slot_runs(name):
    """(slots, idle slots, steps) per run; a step is (positions, effective splits per slot, None if idle)."""
    seq, ns = SHAPES[name][2:]
    L3, L8 = seq // 3, seq // 8
    runs = [(3, (), [((L3 - 1, 0, L3 // 2 + 17), (ns, 1, ns))]),
            (8, (5,), [((0, 63, 64, L8 - 1, L8 // 2 + 5, 0, 64 * ns + 37, 1000), (1, 1, 2, ns, ns, None, ns, ns))])]
    if name == CONSECUTIVE:
        runs.append((3, (1,), [((63, 0, 64), (1, None, 2)), ((64, 0, 65), (2, None, 2))]))
    return runs


def choice_chain(P, j, ns):
    """(effective splits, longest f32 chain in rows, its 32-row tiles) of a choices step: the last split continues over the suffix."""
    n_pos = P + 1
    eff = eff_splits(n_pos, ns)
    chunk = -(-n_pos // eff)
    last = max(0, n_pos - (eff - 1) * chunk)
    return eff, max(chunk, last + j + 1), max(-(-chunk // KTILE), -(-last // KTILE) + -(-(j + 1) // KTILE))


def slot_chain(pos, ns):
    eff = eff_splits(pos + 1, ns)
    chunk = -(-(pos + 1) // eff)
    return eff, chunk, -(-chunk // KTILE)


def test_case_coverage():
    """The case list reaches what the batched steps can get wrong: tile shared memory above 48 KB (bf16 and q80), one split, a
    split count that is not a power of two, the n_splits cap, a slot length that is not a multiple of 64, rotary positions >= 65536
    and the Llama-3.3-70B W2 batch of 8 as two launches; every pinned split count is the mirror's, every step fits the cache."""
    from distributed_llama_b200.ops import gemv_q40_plan
    smem = {False: 0, True: 0}
    effs, capped, odd_slot, max_rot = set(), set(), False, 0
    for name in NAMES:
        nh, nkv, hd, dim, ff = geometry(name)
        seq, ns = SHAPES[name][2:]
        for B, P, js, inactive, eff in choice_runs(name):
            assert eff_splits(P + 1, ns) == eff, (name, B, P)
            assert P + 1 + B * C_OWN <= seq and all(j < C_OWN for j in js) and all(b < B for b in inactive)
            for q8 in smem:
                smem[q8] = max(smem[q8], tile_smem(hd, q8, pow2(B) * nh // nkv))
                assert tile_smem(hd, q8, pow2(B) * nh // nkv) <= SMEM_MAX
            effs.add(eff)
            if eff == ns and P + 1 > 64 * ns:
                capped.add(name)
            max_rot = max(max_rot, P + 1 + max(js))
        for n, idle, steps in slot_runs(name):
            L = seq // n
            odd_slot |= L % 64 != 0
            for pos, want in steps:
                for b in range(n):
                    assert (want[b] is None) == (b in idle)
                    if b not in idle:
                        assert 0 <= pos[b] < L and eff_splits(pos[b] + 1, ns) == want[b], (name, n, pos)
                        effs.add(want[b])
                        if want[b] == ns and pos[b] + 1 > 64 * ns:
                            capped.add(name)
    assert smem[False] > SMEM_DEFAULT and smem[True] > SMEM_DEFAULT, smem
    assert 1 in effs and any(e & (e - 1) for e in effs) and capped == set(NAMES), (effs, capped)
    assert odd_slot and max_rot >= 65536
    _, _, _, dim, ff = geometry("llama-3.3-70b")
    assert any(B == 8 for B, *_ in choice_runs("llama-3.3-70b"))
    for sms in (132, 114):
        p = gemv_q40_plan(PLAIN, RESID, 8, dim, ff, num_sms=sms)
        assert p.rc == 0 and p.launches == 2, p


# ------------------------------------------------------------------ float64 attention of the tile kernels ------------------------------------------------------------------
def tile_attention(q, K, V, hd, chain, bound=True, chunk=32768):
    """float64 softmax(q K^T / sqrt(hd)) V of the query rows q [g, hd] (the kernel's rotated q) over the rows K, V [n, hd] that the
    tile kernel reads, in chunks of rows, and its bound from the kernels' order of operations. chain = (eff, rows, tiles) of the
    longest split. Scores: q pre-scaled by rsqrtf(hd) (2 ulps) and a sequential per-lane sum of hd products, (hd + 10) U sum |q k|.
    Weights: __expf (2 ulps + 1.2 |x| ulps) of the score less the running maximum, then of every rescale of the running maximum
    (at most one per tile) and of the merge weight; the arguments add up to at most s_max - s. acc: one f32 chain over the rows and
    tiles of a split (+ the choice's suffix), then eff merge terms; l: a 5-step warp sum and one update per tile, eff merge terms,
    one division. Returns (z [g, hd], bound [g, hd])."""
    eff, rows, tiles = chain
    c = 1 / math.sqrt(hd)
    n = K.shape[0]
    parts = range(0, n, chunk)
    s = torch.cat([q @ K[r:r + chunk].T for r in parts], 1) * c
    p = torch.softmax(s, -1)
    z = sum(p[:, r:r + chunk] @ V[r:r + chunk] for r in parts)
    if not bound:
        return z, None
    dots = torch.cat([q.abs() @ K[r:r + chunk].abs().T for r in parts], 1) * c
    delta = U * ((hd + 10) * dots + 4 * (tiles + 3) + 3 * (s.amax(-1, keepdim=True) - s))
    pd = p * delta
    e1 = sum(torch.einsum("gp,gpd->gd", pd[:, r:r + chunk], (V[None, r:r + chunk] - z[:, None]).abs()) for r in parts)
    e2 = sum(p[:, r:r + chunk] @ V[r:r + chunk].abs() for r in parts)
    tiny = torch.finfo(torch.float32).tiny      # a q80 value of 0 over one row: z = 0 exactly, and so is the rest of the bound
    return z, e1 + U * (rows + 2 * tiles + eff + 8) * e2 + U * (2 * tiles + eff + 16) * z.abs() + tiny


def attend(q, K, V, hd, chain, bound=True):
    """tile_attention of every KV head: q [nh, hd], K, V [nKv, n, hd] -> (z [nh * hd], bound or None)."""
    nkv = K.shape[0]
    g = q.shape[0] // nkv
    zs, bs = [], []
    for h in range(nkv):
        z, b = tile_attention(q[h * g:(h + 1) * g], K[h], V[h], hd, chain, bound)
        zs.append(z)
        bs.append(b)
    return torch.cat(zs).reshape(-1), (torch.cat(bs).reshape(-1) if bound else None)


# ------------------------------------------------------------------ caches ------------------------------------------------------------------
def cache_view(kv_type, k, v, ks, vs, b=None, L=None):
    """Layer 0's K/V planes as check_kv_rows and kv_of take them: the whole cache, or slot b ([nKv][L][hd] at element b * nKv * L * hd
    of the values, b * nKv * L * hd / 32 of the q80 scales)."""
    if b is not None:
        nkv, _, hd = k.shape
        S = nkv * L * hd
        k, v = (x.view(-1)[b * S:(b + 1) * S].view(nkv, L, hd) for x in (k, v))
        if ks is not None:
            ks, vs = ks[b * S // 32:(b + 1) * S // 32], vs[b * S // 32:(b + 1) * S // 32]
    return types.SimpleNamespace(kv_cache_float_type=kv_type, k_cache=[k], v_cache=[v], k_scale=[ks], v_scale=[vs])


def engine_view(eng, b=None, L=None):
    return cache_view(eng.kv_cache_float_type, eng.k_cache[0], eng.v_cache[0], eng.k_scale[0], eng.v_scale[0], b, L)


def caches_view(eng, caches, b=None, L=None):
    """The random caches as loaded, before any NaN."""
    q8 = eng.kv_cache_float_type == "q80"
    return cache_view(eng.kv_cache_float_type, caches[0][0], caches[1][0], caches[2][0] if q8 else None, caches[3][0] if q8 else None,
                      b, L)


def kv_of(c, idx):
    """Rows idx of a view as the tile kernels multiply them, f64 [nKv, n, hd]: bf16 as stored, q80 int8 x f16 scale (exact in f32)."""
    out = []
    for vals, sc in ((c.k_cache[0], c.k_scale[0]), (c.v_cache[0], c.v_scale[0])):
        assert 0 <= min(idx) and max(idx) < vals.shape[1], "rows outside the view"
        idx = torch.as_tensor(idx, device=vals.device)
        x = vals[:, idx].double()
        if sc is not None:
            nkv, _, hd = vals.shape
            s = _scale_rows(c, sc)[:, idx].double()
            x = (x.view(nkv, -1, hd // 32, 32) * s[..., None]).view(nkv, -1, hd)
        out.append(x)
    return out


def poison(c, ranges):
    """NaN in the bf16 values, or the q80 scales, of the rows [r0, r1) of a view."""
    for vals, sc in ((c.k_cache[0], c.k_scale[0]), (c.v_cache[0], c.v_scale[0])):
        for r0, r1 in ranges:
            if sc is None:
                vals[:, r0:r1] = float("nan")
            else:
                _scale_rows(c, sc)[:, r0:r1] = float("nan")


def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def snapshot(eng):
    return [t.clone() for t in (eng.k_cache[0], eng.v_cache[0], eng.k_scale[0], eng.v_scale[0]) if t is not None]


def check_untouched(eng, before, written, L=None, tag=""):
    """Every cache row but the written ones ((slot or None, row) pairs) is bitwise what it was before the step: NaN rows stay NaN,
    inactive and padding rows write nothing."""
    kv = eng.kv_cache_float_type
    want = [t.clone() for t in before]
    ws = want + [None] * (4 - len(want))
    for b, row in written:
        src, dst = engine_view(eng, b, L), cache_view(kv, *ws, b, L)
        for d, s in ((dst.k_cache[0], src.k_cache[0]), (dst.v_cache[0], src.v_cache[0])):
            d[:, row] = s[:, row]
        if kv == "q80":
            for d, s in ((dst.k_scale[0], src.k_scale[0]), (dst.v_scale[0], src.v_scale[0])):
                _scale_rows(dst, d)[:, row] = _scale_rows(src, s)[:, row]
    for w, t in zip(want, snapshot(eng)):
        assert torch.equal(_bits(w), _bits(t)), f"{tag}: a cache row the step must not write changed"


# ------------------------------------------------------------------ models and engines ------------------------------------------------------------------
@pytest.fixture(scope="module")
def model(request, tmp_path_factory):
    """name -> the 1-layer synthetic model, its device weights and its float64 reference; one model at a time."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    name = request.param
    preset, vocab, seq, _ = SHAPES[name]
    cfg = dataclasses.replace(get_config(preset), n_layers=1, max_seq_len=seq, vocab_size=vocab)
    path = str(tmp_path_factory.mktemp("batched_steps") / f"{name}.m")
    t0 = time.time()
    write_synthetic_model(path, cfg, seed=61, attn_gain=2.0)
    w = load_device_weights(ModelFile(path))
    R = Ref(path)
    print(f"\n[{name}] model ready in {time.time() - t0:.1f} s")
    yield dict(name=name, cfg=cfg, weights=w, ref=R)
    del w, R
    gc.collect()
    torch.cuda.empty_cache()


def _tok(vocab, b, step):
    return (7919 * (b + 1) + 104729 * step + 11) % vocab


def run_step(M, eng, nb, fwd, active, tag):
    """fwd() with W2's block scales zeroed (its final residual is x1), then as is. Returns (scratch, x1, x2, logits) of the nb rows;
    the active rows' scratch must be bitwise that of the zeroed run and free of NaN."""
    w2 = M["weights"].layers[0].w2
    saved = w2.scales.clone()
    w2.scales.zero_()
    try:
        fwd()
        torch.cuda.synchronize()
        I1 = eng.prefill_intermediates(nb, False)
        x1 = eng.x[:nb].double().clone()
    finally:
        w2.scales.copy_(saved)
    fwd()
    torch.cuda.synchronize()
    assert not eng.mega_active, f"{tag}: the step ran the persistent kernel"
    I = eng.prefill_intermediates(nb, False)
    x2, logits = eng.x[:nb].double().clone(), eng.logits[:nb].clone()
    rows = [b for b in range(nb) if b < len(active) and active[b]]
    for k in I:
        assert torch.equal(I1[k][rows], I[k][rows]), f"{tag}: {k} depends on W2's weights"
        assert not torch.isnan(I[k][rows]).any(), f"{tag}: NaN in {k}"
    assert torch.isfinite(x2[rows]).all() and torch.isfinite(logits[rows]).all(), f"{tag}: non-finite residual or logits"
    return I, x1, x2, logits


def same_outputs(eng, nb, rows, ref, tag):
    """The active rows' scratch, residual and logits are bitwise those of `ref` = (scratch, x2, logits)."""
    I = eng.prefill_intermediates(nb, False)
    for k in I:
        assert torch.equal(I[k][rows], ref[0][k][rows]), f"{tag}: {k}"
    assert torch.equal(eng.x[rows].double(), ref[1][rows]) and torch.equal(eng.logits[rows], ref[2][rows]), tag


# ------------------------------------------------------------------ stage checks ------------------------------------------------------------------
def check_step(M, st, tag, rows, I, x1k, x2k, logits):
    """Stage checks of the active rows of one batched step. A row: b, tok, rot (rotary position), view and crow (where its K/V row
    went), idx (the rows it attends to in its view), chain, and controls(): (name, K, V) row sets it must not have attended to."""
    R, L = M["ref"], M["ref"].layers[0]
    hd, nh, nkv, qd, kvd = R.hd, R.nh, R.nkv, R.q_dim, R.kv_dim
    bs = [r["b"] for r in rows]
    x0 = {r["b"]: R.embedding(r["tok"]) for r in rows}
    qkv = I["qkv"].double()
    acts = [q80(rms(x0[b], L["norm0"], R.eps), normed=True) for b in bs]
    kv = gemv_rows(L["qkv"][qd:], acts, gots=[qkv[b, qd:] for b in bs])
    qq = gemv_rows(L["qkv"][:qd], acts)
    for r, (ykv, bkv), (yq, bq) in zip(rows, kv, qq):
        b, rot = r["b"], r["rot"]
        st.r(f"{tag} qkv k|v", ratio(qkv[b, qd:], ykv, bkv))
        q_ref, q_b = norm_rope(yq.view(1, nh, hd), bq.view(1, nh, hd), L["q_norm"], R.rope[rot:rot + 1], R.eps)
        st.r(f"{tag} q (norm+rope)", ratio(qkv[b, :qd].view(1, nh, hd), q_ref, q_b))
        k, v = kv_rows(R, L, qkv[b], R.rope[rot])
        kn = qkv[b, qd:qd + kvd].view(nkv, hd)
        if L["k_norm"] is not None:
            kn = rms(kn, L["k_norm"], R.eps)
        check_kv_rows(r["view"], st, tag, r["crow"], k[None], kn[None], v[None])
        if r["crow"] != rot:
            got, _ = kv_of(r["view"], [r["crow"]])
            kbad = rope(kn, R.rope[r["crow"]])
            if r["view"].k_scale[0] is None:
                unit = bf16_ulp(kbad)
            else:
                unit = 0.5 * _scale_rows(r["view"], r["view"].k_scale[0])[:, r["crow"]].double().repeat_interleave(32, -1)
            st.c("K row rotated for its cache row", float(((got[:, 0] - kbad).abs() / unit).amax()))
        q = qkv[b, :qd].view(nh, hd)
        K, V = kv_of(r["view"], r["idx"])
        z, zb = attend(q, K, V, hd, r["chain"])
        st.r(f"{tag} attention", ratio(I["z"][b], z, zb))
        for name, K2, V2 in r["controls"]():
            z2, _ = attend(q, K2, V2, hd, r["chain"], bound=False)
            st.c(name, ratio(I["z"][b], z2, zb))
    # WO residual from the kernel's attention output
    wo = gemv_rows(L["wo"], [q80(I["z"][b].double()) for b in bs], gots=[x1k[b] - x0[b] for b in bs])
    bound = {}
    for b, (y, bd) in zip(bs, wo):
        x1 = x0[b] + y
        bound[b] = bd + U * x1.abs()
        st.r(f"{tag} wo+residual", ratio(x1k[b], x1, bound[b]))
    for i in range(len(bs) - 1):
        b = bs[i]
        st.c("WO residual from row b+1", float(((x1k[b] - x0[b] - wo[i + 1][0]).abs() / bound[b]).amax()))
    # W1|W3 + SwiGLU, W2 residual, logits
    w13 = gemv_rows(L["w13"], [q80(rms(x1k[b], L["norm1"], R.eps), normed=True) for b in bs])
    for b, (y13, b13) in zip(bs, w13):
        g, u = y13[0::2], y13[1::2]
        sg = torch.sigmoid(g)
        hh = silu(g) * u
        b_h = (sg * (1 + g * (1 - sg))).abs() * u.abs() * b13[0::2] + silu(g).abs() * b13[1::2] + (16 + 2 * g.abs()) * U * hh.abs()
        st.r(f"{tag} w13+swiglu", ratio(I["h"][b], hh, b_h))
    w2 = gemv_rows(L["w2"], [q80(I["h"][b].double()) for b in bs], gots=[x2k[b] - x1k[b] for b in bs])
    for b, (y2, b2) in zip(bs, w2):
        x2 = x1k[b] + y2
        st.r(f"{tag} w2+residual", ratio(x2k[b], x2, b2 + U * x2.abs()))
    lg = gemv_rows(R.wcls, [q80(rms(x2k[b], R.final_norm, R.eps), normed=True) for b in bs], gots=[logits[b] for b in bs])
    for b, (y, bd) in zip(bs, lg):
        st.r(f"{tag} logits", ratio(logits[b], y, bd))
    for i in range(len(bs) - 1):
        st.c("logits of row b+1", float(((logits[bs[i]].double() - lg[i + 1][0]).abs() / lg[i][1]).median()))


def run_choices(M, eng, st, caches, run, tag):
    from distributed_llama_b200.ops import gemv_q40_plan
    B, P, js, inactive, eff_want = run
    R, vocab, (seq, ns) = M["ref"], M["cfg"].vocab_size, SHAPES[M["name"]][2:]
    C, nb, kv_mul = C_OWN, pow2(B), R.nh // R.nkv
    active = [b not in inactive for b in range(B)]
    _load(eng, caches)
    whole, orig = engine_view(eng), caches_view(eng, caches)
    ranges = [(P + 1 + b * C, P + 1 + (b + 1) * C) if b in inactive else (P + 1 + b * C + js[0], P + 1 + (b + 1) * C) for b in range(B)]
    poison(whole, ranges + [(P + 1 + B * C, seq)])
    for j in js:
        t = f"{tag} choices B={B} P={P} j={j}"
        k = f"{tag} choices"
        eff, rows_, tiles = choice_chain(P, j, ns)
        assert eff == eff_want, t
        Rq = nb * kv_mul
        smem = tile_smem(R.hd, eng.kv_cache_float_type == "q80", Rq)
        assert smem <= SMEM_MAX
        w2_launches = gemv_q40_plan(PLAIN, RESID, nb, R.dim, R.ff, num_sms=eng.num_sms).launches
        assert w2_launches == (2 if (M["name"], nb) == ("llama-3.3-70b", 8) else 1), t
        print(f"[{t}] eff {eff}, R {Rq}, tile smem {smem} B, W2 launches {w2_launches}")
        toks = [_tok(vocab, b, j) for b in range(B)]
        before = snapshot(eng)
        I, x1k, x2k, logits = run_step(M, eng, nb, lambda: eng.choices_forward(toks, P, C, j, active), active, t)
        check_untouched(eng, before, [(None, P + 1 + b * C + j) for b in range(B) if active[b]], tag=t)
        act = [b for b in range(B) if active[b]]
        if inactive:
            alt = [tk + 1 if b in inactive else tk for b, tk in enumerate(toks)]
            eng.choices_forward(alt, P, C, j, active)
            torch.cuda.synchronize()
            same_outputs(eng, nb, act, (I, x2k, logits), f"{t}: an inactive choice's token changed an active row")

        def row(b):
            own = list(range(P + 1 + b * C, P + 1 + b * C + j + 1))
            idx = list(range(P + 1)) + own

            def controls():
                out = [("attention without the new row", *kv_of(whole, idx[:-1]))]
                if own[-1] + 1 < seq:
                    K, V = kv_of(whole, idx)
                    K1, V1 = kv_of(orig, [own[-1] + 1])
                    out.append(("attention one row past the new row", torch.cat([K, K1], 1), torch.cat([V, V1], 1)))
                if b + 1 < B and active[b + 1]:
                    out.append(("choice b attending to choice b+1's rows", *kv_of(whole, list(range(P + 1)) + [x + C for x in own])))
                return out
            return dict(b=b, tok=toks[b], rot=P + 1 + j, view=whole, crow=own[-1], idx=idx, chain=(eff, rows_, tiles), controls=controls)
        check_step(M, st, k, [row(b) for b in act], I, x1k, x2k, logits)


def run_slots(M, eng, st, caches, run, tag, alone=False):
    n, idle, steps = run
    R, vocab, (seq, ns) = M["ref"], M["cfg"].vocab_size, SHAPES[M["name"]][2:]
    eng.set_slots(n)
    L, nb, kv_mul = eng.slot_len, pow2(n), R.nh // R.nkv
    assert L == seq // n
    active = [b not in idle for b in range(n)]
    act = [b for b in range(n) if active[b]]
    _load(eng, caches)
    views = [engine_view(eng, b, L) for b in range(n)]
    origs = [caches_view(eng, caches, b, L) for b in range(n)]
    for b in range(n):
        poison(views[b], [(0, L)] if b in idle else [(steps[0][0][b], L)])
    for i, (pos, effs) in enumerate(steps):
        t, k = f"{tag} slots n={n} pos={pos}", f"{tag} slots"
        smem = tile_smem(R.hd, eng.kv_cache_float_type == "q80", kv_mul)
        assert smem <= SMEM_DEFAULT
        print(f"[{t}] eff {effs}, R {kv_mul}, tile smem {smem} B")
        toks = [_tok(vocab, b, 1000 + i) for b in range(n)]
        before = snapshot(eng)
        I, x1k, x2k, logits = run_step(M, eng, nb, lambda: eng.slots_forward(toks, pos, active), active, t)
        check_untouched(eng, before, [(b, pos[b]) for b in act], L, tag=t)
        if idle:
            alt = [tk + 1 if b in idle else tk for b, tk in enumerate(toks)]
            eng.slots_forward(alt, pos, active)
            torch.cuda.synchronize()
            same_outputs(eng, nb, act, (I, x2k, logits), f"{t}: an idle slot's token changed an active row")
        if alone:
            for b in act:
                lg = eng.slots_forward(toks, pos, [c == b for c in range(n)])
                assert torch.equal(lg[b], logits[b]), f"{t}: slot {b} alone differs from the batched step"

        def row(b):
            p = pos[b]
            eff, rows_, tiles = slot_chain(p, ns)
            assert eff == effs[b], t
            idx = list(range(p + 1))

            def controls():
                out = []
                if p > 0:
                    out.append(("attention without the new row", *kv_of(views[b], idx[:-1])))
                if p + 1 < L:
                    K, V = kv_of(views[b], idx)
                    K1, V1 = kv_of(origs[b], [p + 1])
                    out.append(("attention one row past the new row", torch.cat([K, K1], 1), torch.cat([V, V1], 1)))
                if b + 1 < n:
                    out.append(("slot b attending to slot b+1's rows", *kv_of(origs[b + 1], idx)))
                return out
            return dict(b=b, tok=toks[b], rot=p, view=views[b], crow=p, idx=idx, chain=(eff, rows_, tiles), controls=controls)
        check_step(M, st, k, [row(b) for b in act], I, x1k, x2k, logits)
    eng.set_slots(1)


@pytest.mark.gpu
@pytest.mark.parametrize("model", NAMES, indirect=True)
def test_batched_steps_against_float64(model):
    """Every stage of every active row of the choices and slots steps against float64 from the engine's own input to that stage,
    with both cache types; cache rows, NaN sentinels, inactive rows and negative controls."""
    from distributed_llama_b200.runtime import Engine
    name = model["name"]
    ns = SHAPES[name][3]
    st = Stats()
    t0 = time.time()
    for kv in ("bf16", "q80"):
        eng = Engine(model["weights"], n_splits=ns, kv_cache_float_type=kv)
        assert eng.n_splits == ns and eng.max_batch == 8
        caches = _random_caches(eng, 2026)
        for run in choice_runs(name):
            run_choices(model, eng, st, caches, run, f"{name} {kv}")
        for run in slot_runs(name):
            run_slots(model, eng, st, caches, run, f"{name} {kv}", alone=name == ALONE and run[0] == 8)
        del eng, caches
        gc.collect()
        torch.cuda.empty_cache()
    print(f"\n[{name}] {time.time() - t0:.1f} s")
    st.report(name)


# ------------------------------------------------------------------ kernel sweep ------------------------------------------------------------------
SWEEP_SEQ = 4096


def _sweep_cache(shape, q8, g):
    if not q8:
        return torch.randn(shape, generator=g, device="cuda").bfloat16(), None
    vals = torch.randint(-127, 128, shape, generator=g, device="cuda", dtype=torch.int8)
    sc = (torch.rand(shape[0] * shape[1] * shape[2] // 32 + 8, generator=g, device="cuda") * 0.01 + 0.005).half()
    return vals, sc


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "q80"])
def test_tile_kernels_sweep(kv):
    """dl_choice_attn_only and dl_slot_attn alone at every (heads, kv heads, head dim) of the shapes, B 1, 3 and 8 (one inactive
    row of 8), P + 1 and pos + 1 either side of the split-count steps at 64 and 64 * n_splits, against tile_attention."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    q8 = kv == "q80"
    st = Stats()
    for name in NAMES:
        nh, nkv, hd, _, _ = geometry(name)
        ns = SHAPES[name][3]
        kv_mul, q_dim = nh // nkv, nh * hd
        qkv_dim = q_dim + 2 * nkv * hd
        g = torch.Generator(device="cuda").manual_seed(len(name) * 1009 + hd + q8)
        kc, ks = _sweep_cache((nkv, SWEEP_SEQ, hd), q8, g)
        vc, vs = _sweep_cache((nkv, SWEEP_SEQ, hd), q8, g)
        whole = cache_view(kv, kc, vc, ks, vs)
        for B in (1, 3, 8):
            mask = 1 << 2 if B == 8 else 0
            qkv = torch.randn(B, qkv_dim, generator=g, device="cuda") * 2.0
            partial = torch.full((B * nh * ns * (hd + 2),), float("nan"), device="cuda")
            # choices: P + 1 at 64, 65, 64 * ns and 64 * ns + 1 rows
            C = 40
            j = {1: 0, 3: C - 1, 8: 17}[B]
            for P in (63, 64, 64 * ns - 1, 64 * ns):
                counters = torch.zeros(nkv, dtype=torch.int32, device="cuda")
                out = torch.full((B, q_dim), float("nan"), device="cuda")
                args = [qkv.data_ptr(), qkv_dim, kc.data_ptr(), vc.data_ptr()]
                if q8:
                    args += [ks.data_ptr(), vs.data_ptr()]
                args += [nh, nkv, hd, SWEEP_SEQ, ns, B, P, C, j, mask, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim,
                         cl.stream_ptr()]
                rc = (lib.dl_choice_attn_only_q80 if q8 else lib.dl_choice_attn_only)(*args)
                assert rc == 0, (name, B, P)
                torch.cuda.synchronize()
                assert int(counters.abs().sum()) == 0
                chain = choice_chain(P, j, ns)
                for b in range(B):
                    if (mask >> b) & 1:
                        continue
                    idx = list(range(P + 1)) + list(range(P + 1 + b * C, P + 2 + b * C + j))
                    K, V = kv_of(whole, idx)
                    z, zb = attend(qkv[b, :q_dim].double().view(nh, hd), K, V, hd, chain)
                    st.r(f"{kv} choice kernel", ratio(out[b], z, zb))
            # slots: B slots of L rows, positions either side of the split-count steps
            L = SWEEP_SEQ // B
            cands = [63, 64, 64 * ns - 1, 64 * ns, L - 1, 0, 1000, 64 * ns + 37]
            pos = [min(cands[(b + B) % len(cands)], L - 1) for b in range(B)]
            counters = torch.zeros(B * nkv, dtype=torch.int32, device="cuda")
            out = torch.full((B, q_dim), float("nan"), device="cuda")
            posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
            args = [qkv.data_ptr(), qkv_dim, posd.data_ptr(), kc.data_ptr(), vc.data_ptr()]
            if q8:
                args += [ks.data_ptr(), vs.data_ptr()]
            args += [nh, nkv, hd, L, ns, B, mask, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, cl.stream_ptr()]
            assert (lib.dl_slot_attn_q80 if q8 else lib.dl_slot_attn)(*args) == 0, (name, B)
            torch.cuda.synchronize()
            assert int(counters.abs().sum()) == 0
            for b in range(B):
                if (mask >> b) & 1:
                    continue
                K, V = kv_of(cache_view(kv, kc, vc, ks, vs, b, L), list(range(pos[b] + 1)))
                z, zb = attend(qkv[b, :q_dim].double().view(nh, hd), K, V, hd, slot_chain(pos[b], ns))
                st.r(f"{kv} slot kernel", ratio(out[b], z, zb))
            del qkv, partial
    st.report(f"{kv} sweep")
