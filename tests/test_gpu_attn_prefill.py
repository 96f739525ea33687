"""Prompt-chunk attention on the tensor cores (attnPrefillTcKernel, csrc/cuda/attn_prefill_tc.cu) and its per-token fallback
(attnDecodeKernel with one split, as the engine runs it under DL_NO_TC_ATTN=1) against float64 references, for bf16 and q80 caches.

Reference. The tensor-core path is compared with float64 attention over exactly the operands the tensor cores see:
* q~ = bf16(f32(q) * f32(log2(e) / sqrt(hd))), rounded like apPack;
* K and V as stored; for q80 the widened tile bf16(f32(int8) * f32(f16 scale)) that apWidenTile produces (not the exact value);
* out = softmax_2(q~ . K^T) . V over positions 0 .. p0 + t, for every (token t, head).
The fallback is compared with float64 softmax(q . K^T / sqrt(hd)) . V over the unrounded q and the exact dequantised cache.

Bound, per (token, head) row. The steps the tensor-core reference does not mirror are:
* P = exp2(S - m) rounded to bf16 before P.V, a relative error of at most 2^-9 per weight. The normaliser l sums the unrounded
  weights, so the output moves by at most 2^-9 * sum(p |V|) / l <= 2^-9 * max|V| over the row's visible positions;
* exp2f (ex2.approx, relative error below 2^-22), the f32 scores of the wgmma and the f32 sums of l and O: each weight moves by a
  relative 1e-5 or less at these scores, about 2^-17; the bound gives them 2^-14 * max|V|;
* the bf16 output: half an ulp of the computed value, at most one bf16 ulp of the reference.
So the tensor-core bound is (2^-9 + 2^-14) * max|V_visible| + bf16_ulp(ref). The fallback keeps f32 weights and gets the decode
bound of test_gpu_decode_attn.py, 2e-4 * max|V_visible| + bf16_ulp(ref).
On an H100 80GB HBM3 (700 W power limit) the largest error over all cases is 0.55 of the bound on the tensor-core path and 0.49
on the fallback. Most of either is the rounding of the bf16 output, which alone reaches 0.5.

Inputs. Scores have a standard deviation of about 4 (q * 4 against unit keys), so softmaxes are peaked, not flat. Needle keys
parallel to q~ of a chosen (token, head), at score 30, sit on the row's diagonal p0 + t and one position past it (which must stay
masked), for the rows whose diagonal is at KV-tile positions 63 / 64 and 127 / 128, for the first and last token of query tiles
and for the packed rows 63 / 64 where the two consumer warpgroups split a tile. Eight keys at score 22 in an earlier KV tile (or
half-tile) than the needle make pass 1 rescale l.

Shapes (nHeads / nKvHeads / headDim) cover GQA packings of 1 to 128 heads per KV head, with 128-row tiles, 126-row (kvMul 3)
and 125-row (kvMul 5) tiles, and one-token tiles of 96 and 128 rows. Positions cover single tokens at a tile edge, T = tq and
tq + 1 for the shape, the default 192-token chunking (the second chunk starts mid-tile), chunks ending on and one past a
128-row tile, a chunk ending at the last row of a 1000-row cache, and a 256-token chunk at position 16128.

How far a broken kernel lands (worst err / bound over the tensor-core cases, H100, each mutation run once):
* causal mask `<` instead of `<=` (drops the diagonal): 500x;
* causal mask `<= rowPos + 1` (sees one key too many): 760x;
* token of a packed row as `row % kvMul` instead of `row / kvMul`: 760x;
* pass 1 without the exp2f(m - mNew) rescale of l: 155x;
* q scaled by 1 / sqrt(hd) instead of log2(e) / sqrt(hd): 84x.
Contracts: the kernel reads no cache row outside [0, p0 + T) of its own head (the others hold NaN) and nothing outside its slot,
writes nothing but its output columns, gives bitwise equal results on repeated launches and refuses unsupported shapes without
launching. The 454 tests of this file run in 17 s on that H100.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from test_gpu_decode_attn import bf16_ulp
from test_gpu_kv_q80 import q80_quant

LOG2E = 1.4426950408889634
NEEDLE_SCORE = 30.0     # natural-log score of a needle key against its row's q
MODERATE_SCORE = 22.0   # the earlier block that pass 1 has to rescale
N_MODERATE = 8
TOL_TC = 2.0 ** -9 + 2.0 ** -14   # tensor-core bound, in units of max|V| over the visible rows
TOL_FALLBACK = 2e-4               # fallback (f32 weights) bound, the same units
CACHES = ("bf16", "q80")


# ---- float64 reference and needle construction (CPU or CUDA tensors) ----------------------------------------------------------
def scale_log2(hd: int) -> torch.Tensor:
    """The f32 factor the launcher folds into q: log2(e) / sqrtf(hd), both rounded to f32 on the host."""
    return torch.tensor(LOG2E, dtype=torch.float32) / torch.sqrt(torch.tensor(float(hd), dtype=torch.float32))


def q_tensor_core(q: torch.Tensor, hd: int) -> torch.Tensor:
    """q [..., hd] f32 -> the bf16 q~ that the kernel stores for the wgmma: bf16(f32(q) * f32 scale), round to nearest even."""
    return (q.float() * scale_log2(hd).to(q.device)).bfloat16()


def ref_prefill(q: torch.Tensor, K: torch.Tensor, V: torch.Tensor, p0: int, c: float, max_elems: int = 1 << 24) -> torch.Tensor:
    """softmax(c * q . K^T) . V of token t over positions 0 .. p0 + t, per head; q-head h reads KV head h // (nHeads / nKvHeads).
    q [T, nHeads, hd]; K, V [nKvHeads, >= p0 + T, hd]. c = ln 2 for the base-2 scores of q~, 1 / sqrt(hd) for a plain q.
    Returns f64 [T, nHeads, hd]; works per KV head and in token blocks of at most max_elems scores."""
    T, n_heads, hd = q.shape
    n_kv = K.shape[0]
    g = n_heads // n_kv
    P = p0 + T
    dev = q.device
    qd = q.double().view(T, n_kv, g, hd)
    hidden = torch.arange(P, device=dev)[None, :] > (p0 + torch.arange(T, device=dev))[:, None]   # [T, P]
    step = max(1, max_elems // (g * P))
    out = torch.empty(T, n_heads, hd, dtype=torch.float64, device=dev)
    for kvh in range(n_kv):
        Kh, Vh = K[kvh, :P].double(), V[kvh, :P].double()
        for t0 in range(0, T, step):
            s = torch.einsum("tgd,pd->tgp", qd[t0:t0 + step, kvh], Kh) * c
            s.masked_fill_(hidden[t0:t0 + step, None, :], float("-inf"))
            out[t0:t0 + step, kvh * g:(kvh + 1) * g] = torch.einsum("tgp,pd->tgd", torch.softmax(s, dim=-1), Vh)
    return out


def visible_vmax(V: torch.Tensor, p0: int, T: int, kv_mul: int) -> torch.Tensor:
    """max|V| over the positions 0 .. p0 + t that token t sees, per (token, head): f64 [T, nHeads]."""
    rowmax = V[:, :p0 + T].double().abs().amax(dim=-1)                 # [nKv, P]
    return torch.cummax(rowmax, dim=1).values[:, p0:].T.repeat_interleave(kv_mul, dim=1)


def needle_plan(T: int, p0: int, seq: int, n_heads: int, n_kv: int):
    """Keys to plant: {(kvh, position): (t, h, natural score)}, parallel to q~ of row (t, h). Earlier entries win a position.
    Rows: diagonals at KV-tile positions 63 / 64 / 127 / 128 (mod 128), the first and last token of the first, second and last
    query tile, and the packed rows 63 / 64 of the first and last query tile. Each row gets a needle on its diagonal and one
    position past it, and a block of moderate keys in the KV tile (or half-tile) before its diagonal."""
    kv_mul = n_heads // n_kv
    tq = 128 // kv_mul
    n_tiles = -(-T // tq)
    rows = [(t, (3 * t + 1) % n_heads) for t in range(T) if (p0 + t) % 64 in (0, 63)]
    for qt in sorted({0, 1, n_tiles - 1} & set(range(n_tiles))):
        t0 = qt * tq
        rows += [(t, (3 * t + 1) % n_heads) for t in (t0, min(t0 + tq, T) - 1)]
        if qt in (0, n_tiles - 1):
            for r in (63, 64):
                t = t0 + r // kv_mul
                if r // kv_mul < tq and t < T:
                    rows.append((t, (t % n_kv) * kv_mul + r % kv_mul))
    seen = set()
    rows = [r for r in rows if not (r in seen or seen.add(r))]
    plan = {}

    def put(h, pos, t, score):
        if 0 <= pos < seq:
            plan.setdefault((h // kv_mul, pos), (t, h, score))
    for t, h in rows:
        put(h, p0 + t, t, NEEDLE_SCORE)
    for t, h in rows:
        put(h, p0 + t + 1, t, NEEDLE_SCORE)
    for t, h in rows:
        d = p0 + t
        start = (d // 128 - 1) * 128 if d >= 128 else (0 if d >= 64 else -1)
        if start >= 0:
            for i in range(N_MODERATE):
                put(h, start + i, t, MODERATE_SCORE)
    return plan


def plant(K: torch.Tensor, q_tc: torch.Tensor, plan) -> None:
    """K [nKv, seq, hd] f32 in place: K[kvh, pos] = q~[t, h] scaled to the base-2 score `score * log2(e)` (natural score `score`)."""
    for (kvh, pos), (t, h, score) in plan.items():
        qv = q_tc[t, h].float()
        K[kvh, pos] = qv * (score * LOG2E / float(qv @ qv))


def test_reference_helpers_on_cpu():
    """The reference against a per-row loop, the per-row max|V|, the q~ rounding, and needles that take their rows' softmax."""
    g = torch.Generator().manual_seed(5)
    n_heads, n_kv, hd, T, p0, seq = 6, 2, 64, 9, 60, 80
    q = torch.randn(T, n_heads, hd, generator=g) * 4
    K = torch.randn(n_kv, seq, hd, generator=g)
    V = torch.randn(n_kv, seq, hd, generator=g)
    q_tc = q_tensor_core(q, hd)
    for d in (64, 128):   # the host's f32 arithmetic
        assert float(scale_log2(d)) == float(np.float32(LOG2E) / np.sqrt(np.float32(d)))
    want = (q.double() * float(scale_log2(hd))).float().bfloat16()   # the product is exact in f64: one rounding to f32, then to bf16
    assert torch.equal(q_tc.view(torch.int16), want.view(torch.int16))
    plan = needle_plan(T, p0, seq, n_heads, n_kv)
    # T = 9 at p0 = 60: diagonals 63 and 64 (t = 3, 4); one query tile of 42 tokens: first and last token; packed rows 63 / 64 lie
    # past T (tokens 21, 21)
    rows = {(t, h) for t, h, s in plan.values() if s == NEEDLE_SCORE}
    assert rows == {(3, 10 % 6), (4, 13 % 6), (0, 1), (8, 25 % 6)}
    assert {pos for (kvh, pos), (t, h, s) in plan.items() if (t, h) == (4, 1)} >= {64, 65, 0}
    plant(K, q_tc, plan)
    for (kvh, pos), (t, h, s) in plan.items():
        assert abs(float(q_tc[t, h].double() @ K[kvh, pos].double()) - s * LOG2E) < 1e-3 * s
    ref = ref_prefill(q_tc, K, V, p0, math.log(2), max_elems=50)        # several token blocks
    vmax = visible_vmax(V, p0, T, 3)
    for t in range(T):
        for h in range(n_heads):
            n = p0 + t + 1
            s = (K[h // 3, :n].double() @ q_tc[t, h].double()) * math.log(2)
            assert torch.allclose(ref[t, h], torch.softmax(s, 0) @ V[h // 3, :n].double(), rtol=0, atol=1e-12)
            assert vmax[t, h].item() == V[h // 3, :n].abs().max().item()
    # a needle row attends to its diagonal key and not to the one past it: its output is V of the diagonal row, up to the
    # weight e^-8 of each of the 8 moderate keys
    for (kvh, pos), (t, h, s) in plan.items():
        if pos == p0 + t and s == NEEDLE_SCORE:
            assert (ref[t, h] - V[kvh, pos].double()).abs().max().item() < 1e-2, (t, h)
    # the unrounded-q reference of the fallback agrees with the base-2 one to the rounding of q
    ref_n = ref_prefill(q, K, V, p0, 1 / math.sqrt(hd))
    assert (ref_n - ref).abs().max().item() < 0.05


# ---- harness ------------------------------------------------------------------------------------------------------------------
def _dequant(q: torch.Tensor, s: torch.Tensor, dtype) -> torch.Tensor:
    """int8 values times their block's f16 scale, both converted to and multiplied in `dtype` (f32: exact, as apWidenTile does)."""
    return (q.to(dtype).view(*q.shape[:-1], -1, 32) * s.to(dtype).unsqueeze(-1)).view(q.shape)


class Cache:
    """A K/V cache [nKv, seq, hd] as the kernels read it: bf16, or q80 int8 values with an f16 scale plane. `kt` / `vt` are what
    the tensor cores see, `kx` / `vx` the exact values the fallback reads."""

    def __init__(self, kind: str, K: torch.Tensor, V: torch.Tensor):
        self.kind = kind
        if kind == "bf16":
            self.k, self.v = K.bfloat16().contiguous(), V.bfloat16().contiguous()
            self.ks = self.vs = None
            self.kt = self.kx = self.k
            self.vt = self.vx = self.v
            return
        (self.k, self.ks), (self.v, self.vs) = q80_quant(K), q80_quant(V)
        self.k, self.v, self.ks, self.vs = self.k.contiguous(), self.v.contiguous(), self.ks.contiguous(), self.vs.contiguous()
        self.kt, self.vt = _dequant(self.k, self.ks, torch.float32).bfloat16(), _dequant(self.v, self.vs, torch.float32).bfloat16()
        self.kx, self.vx = _dequant(self.k, self.ks, torch.float64), _dequant(self.v, self.vs, torch.float64)

    def ptrs(self):
        return (self.k.data_ptr(), self.v.data_ptr(), self.ks.data_ptr() if self.ks is not None else None,
                self.vs.data_ptr() if self.vs is not None else None)

    def poison_rows(self, start: int):
        """Rows [start, seq) of every head hold NaN (q80: their scales)."""
        if self.kind == "bf16":
            self.k[:, start:] = float("nan")
            self.v[:, start:] = float("nan")
        else:
            self.ks[:, start:] = float("nan")
            self.vs[:, start:] = float("nan")


def _inputs(cache, n_heads, n_kv, hd, T, p0, seq):
    """qkv rows [T, q|k|v] with scores of std ~4, needle keys planted, and the cache built from the keys."""
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(repr((cache, n_heads, n_kv, hd, T, p0, seq)).encode()))
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    qkv = torch.randn(T, q_dim + 2 * kv_dim, device="cuda", generator=gen)
    qkv[:, :q_dim] *= 4.0
    K = torch.randn(n_kv, seq, hd, device="cuda", generator=gen)
    V = torch.randn(n_kv, seq, hd, device="cuda", generator=gen)
    q = qkv[:, :q_dim].view(T, n_heads, hd)
    plant(K, q_tensor_core(q, hd), needle_plan(T, p0, seq, n_heads, n_kv))
    return qkv, Cache(cache, K, V)


def _run_tc(qkv, T, p0, n_heads, n_kv, hd, seq, ptrs, out, out_stride):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    k, v, ks, vs = ptrs
    if ks is None and vs is None:
        return lib.dl_attn_prefill_tc(qkv.data_ptr(), qkv.shape[1], T, p0, n_heads, n_kv, hd, seq, k, v, out, out_stride, cl.stream_ptr())
    return lib.dl_attn_prefill_tc_q80(qkv.data_ptr(), qkv.shape[1], T, p0, n_heads, n_kv, hd, seq, k, v, ks, vs, out, out_stride,
                                      cl.stream_ptr())


def _tc(qkv, c, T, p0, n_heads, n_kv, hd, seq, ptrs=None):
    out = torch.full((T, n_heads * hd), float("nan"), dtype=torch.bfloat16, device="cuda")
    rc = _run_tc(qkv, T, p0, n_heads, n_kv, hd, seq, ptrs or c.ptrs(), out.data_ptr(), n_heads * hd)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return out.view(T, n_heads, hd)


def _fallback(qkv, c, T, p0, n_heads, n_kv, hd, seq, ptrs=None):
    """attnDecodeKernel over the chunk as enginePrefill launches it: nb = T, pos[t] = p0 + t, one split, bf16 output."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    k, v, ks, vs = ptrs or c.ptrs()
    q_dim = n_heads * hd
    pos = torch.arange(p0, p0 + T, dtype=torch.int32, device="cuda")
    partial = torch.empty(T * n_heads * (hd + 2), device="cuda")
    counters = torch.zeros(T * n_heads, dtype=torch.int32, device="cuda")
    out = torch.full((T, q_dim), float("nan"), dtype=torch.bfloat16, device="cuda")
    if ks is None:
        rc = lib.dl_attn_decode(qkv.data_ptr(), qkv.shape[1], pos.data_ptr(), k, v, n_heads, n_kv, hd, seq, 1, partial.data_ptr(),
                                counters.data_ptr(), None, q_dim, out.data_ptr(), T, cl.stream_ptr())
    else:
        rc = lib.dl_attn_decode_q80(qkv.data_ptr(), qkv.shape[1], pos.data_ptr(), k, v, ks, vs, n_heads, n_kv, hd, seq, 1,
                                    partial.data_ptr(), counters.data_ptr(), None, q_dim, out.data_ptr(), T, cl.stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert int(counters.abs().sum()) == 0, "split counters not reset"
    return out.view(T, n_heads, hd)


def _ratio(got, ref, vmax, tol_v):
    """Largest err / bound over the elements and the (token, head, column) where it is."""
    assert torch.isfinite(got).all(), f"non-finite output at (token, head, col) {tuple(torch.nonzero(~torch.isfinite(got))[0].tolist())}"
    r = (got.double() - ref).abs() / (tol_v * vmax[..., None] + bf16_ulp(ref))
    i = int(r.argmax())
    return r.view(-1)[i].item(), tuple(int(x) for x in torch.unravel_index(torch.tensor(i), r.shape))


def tc_ratio(cache, n_heads, n_kv, hd, T, p0, seq):
    """Worst err / bound of the tensor-core kernel on one case, and where."""
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, seq)
    got = _tc(qkv, c, T, p0, n_heads, n_kv, hd, seq)
    q = q_tensor_core(qkv[:, :n_heads * hd].view(T, n_heads, hd), hd)
    ref = ref_prefill(q, c.kt, c.vt, p0, math.log(2))
    return _ratio(got, ref, visible_vmax(c.vt, p0, T, n_heads // n_kv), TOL_TC)


def fallback_ratio(cache, n_heads, n_kv, hd, T, p0, seq):
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, seq)
    got = _fallback(qkv, c, T, p0, n_heads, n_kv, hd, seq)
    ref = ref_prefill(qkv[:, :n_heads * hd].view(T, n_heads, hd), c.kx, c.vx, p0, 1 / math.sqrt(hd))
    return _ratio(got, ref, visible_vmax(c.vx, p0, T, n_heads // n_kv), TOL_FALLBACK)


# ---- cases --------------------------------------------------------------------------------------------------------------------
SHAPES = [(32, 8, 128),    # Llama-3.1-8B, Qwen3-8B
          (32, 4, 128),    # Qwen3-30B-A3B
          (16, 8, 128),    # Qwen3-0.6B
          (32, 32, 128),   # Llama-2-7B: tq 128
          (64, 4, 128),    # Qwen3-235B-A22B: tq 8
          (24, 8, 128),    # Llama-3.2-3B: 126-row tiles
          (40, 8, 128),    # 125-row tiles
          (32, 8, 64),     # Llama-3.2-1B
          (96, 1, 64),     # one token, 96 rows
          (128, 1, 128),   # one token, 128 rows
          (6, 2, 64)]
EDGE_SHAPES = [(32, 8, 128), (128, 1, 128), (6, 2, 64)]
EDGE_POSITIONS = [(1, 0), (1, 127), (1, 128), (192, 0), (192, 192), (256, 0), (256, 3840), (100, 28), (101, 28), (256, 744, 1000)]


def _core_positions(n_heads, n_kv):
    tq = 128 // (n_heads // n_kv)
    return [(1, 128), (tq, 0), (tq + 1, 61), (192, 192), (101, 28)]


def _with_seq(pos):
    T, p0 = pos[:2]
    return (T, p0, pos[2] if len(pos) > 2 else p0 + T + 77)   # default: rows past the chunk, not a multiple of 128


def _cases():
    out = []
    for shape in SHAPES:
        for pos in _core_positions(*shape[:2]) + (EDGE_POSITIONS if shape in EDGE_SHAPES else []):
            out += [(cache, *shape, *_with_seq(pos)) for cache in CACHES]
    out += [(cache, 32, 8, 128, 256, 16128, 16384) for cache in CACHES]
    # the cases of the earlier f32-bound tests: bf16 caches of 640 rows, q80 caches of p0 + T + 40 rows
    out += [("bf16", *shape, T, p0, 640) for shape in [(32, 8, 128), (8, 8, 128), (40, 8, 128), (32, 4, 128), (32, 8, 64), (4, 1, 128), (6, 2, 64)]
            for T, p0 in [(64, 0), (5, 0), (33, 100), (200, 0), (192, 300), (1, 7)]]
    out += [("q80", *shape, T, p0, p0 + T + 40) for shape in [(32, 8, 128), (8, 8, 128), (32, 8, 64), (6, 2, 64)]
            for T, p0 in [(1, 7), (63, 100), (64, 0), (192, 300), (256, 5)]]
    return list(dict.fromkeys(out))


CASES = _cases()
_IDS = [f"{c}-{h}/{k}/{d}-T{T}-p{p0}-s{s}" for c, h, k, d, T, p0, s in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("cache,n_heads,n_kv,hd,T,p0,seq", CASES, ids=_IDS)
def test_attn_prefill_tc_matches_float64(cache, n_heads, n_kv, hd, T, p0, seq):
    r, where = tc_ratio(cache, n_heads, n_kv, hd, T, p0, seq)
    assert r <= 1.0, f"err = {r:.3g} x bound at (token, head, col) {where}"


@pytest.mark.gpu
@pytest.mark.parametrize("cache,n_heads,n_kv,hd,T,p0,seq", CASES, ids=_IDS)
def test_attn_prefill_fallback_matches_float64(cache, n_heads, n_kv, hd, T, p0, seq):
    r, where = fallback_ratio(cache, n_heads, n_kv, hd, T, p0, seq)
    assert r <= 1.0, f"err = {r:.3g} x bound at (token, head, col) {where}"


# ---- contracts ----------------------------------------------------------------------------------------------------------------
def _check_both(qkv, c, T, p0, n_heads, n_kv, hd, seq, ptrs=None, what=""):
    """Both paths against their references over the rows [0, p0 + T) of the cache `c` describes."""
    kv_mul = n_heads // n_kv
    q = qkv[:, :n_heads * hd].view(T, n_heads, hd)
    ref = ref_prefill(q_tensor_core(q, hd), c.kt, c.vt, p0, math.log(2))
    r, where = _ratio(_tc(qkv, c, T, p0, n_heads, n_kv, hd, seq, ptrs), ref, visible_vmax(c.vt, p0, T, kv_mul), TOL_TC)
    assert r <= 1.0, f"{what} tensor cores: err = {r:.3g} x bound at {where}"
    ref = ref_prefill(q, c.kx, c.vx, p0, 1 / math.sqrt(hd))
    r, where = _ratio(_fallback(qkv, c, T, p0, n_heads, n_kv, hd, seq, ptrs), ref, visible_vmax(c.vx, p0, T, kv_mul), TOL_FALLBACK)
    assert r <= 1.0, f"{what} fallback: err = {r:.3g} x bound at {where}"


@pytest.mark.gpu
@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("n_heads,n_kv,hd,T,p0,seq", [(32, 8, 128, 101, 28, 300), (32, 8, 128, 192, 192, 1000), (6, 2, 64, 256, 744, 1000),
                                                       (24, 8, 128, 43, 61, 200), (128, 1, 128, 1, 128, 300), (16, 8, 128, 5, 0, 131)])
def test_attn_prefill_reads_only_the_chunk_rows(cache, n_heads, n_kv, hd, T, p0, seq):
    """Every cache row at or past p0 + T of every head holds NaN (q80: its scales): rows not written yet, or a previous request's
    in a reused slot. The output must not depend on them."""
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, seq)
    c.poison_rows(p0 + T)
    _check_both(qkv, c, T, p0, n_heads, n_kv, hd, seq, what="NaN rows past the chunk:")


@pytest.mark.gpu
@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("n_heads,n_kv,hd,T,p0", [(32, 8, 128, 256, 744), (6, 2, 64, 100, 28)])
def test_attn_prefill_slot_addressing(cache, n_heads, n_kv, hd, T, p0):
    """Slot 1 of three 1000-row slots, addressed as the engine does (cache + slot * nKvHeads * slotLen * hd, seqLen = slotLen;
    scales at a 32nd of that offset). Slots 0 and 2 hold NaN."""
    L, slot = 1000, 1
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, L)
    bufs = []
    for x in (c.k, c.v, c.ks, c.vs):
        if x is not None:   # three slots [3][nKv][L][hd] (scales [3][nKv][L][hd / 32]); the other two NaN (int8 values: -128)
            bufs.append(torch.full((3, *x.shape), float("nan") if x.is_floating_point() else -128, dtype=x.dtype, device="cuda"))
            bufs[-1][slot] = x
    ptrs = tuple(b[slot].data_ptr() for b in bufs) + (None, None) * (cache == "bf16")
    _check_both(qkv, c, T, p0, n_heads, n_kv, hd, L, ptrs=ptrs, what=f"slot {slot}:")


SENTINEL = 0x7FA5   # a bf16 quiet NaN with a payload no arithmetic produces


@pytest.mark.gpu
@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("n_heads,n_kv,hd,T,p0", [(24, 8, 128, 43, 61), (96, 1, 64, 3, 126), (32, 8, 64, 33, 100)])
def test_attn_prefill_writes_only_its_columns(cache, n_heads, n_kv, hd, T, p0):
    """outStride = qDim + 64 and one row past the chunk, all set to a NaN sentinel first: only columns [0, qDim) of rows
    [0, T) change; they hold the attention output."""
    seq = p0 + T + 77
    q_dim = n_heads * hd
    stride = q_dim + 64
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, seq)
    out = torch.full(((T + 1) * stride,), SENTINEL, dtype=torch.int16, device="cuda")
    assert _run_tc(qkv, T, p0, n_heads, n_kv, hd, seq, c.ptrs(), out.data_ptr(), stride) == 0
    torch.cuda.synchronize()
    rows = out.view(T + 1, stride)
    assert (rows[:T, q_dim:] == SENTINEL).all() and (rows[T] == SENTINEL).all(), "written outside the output columns"
    got = rows[:T, :q_dim].view(torch.bfloat16).view(T, n_heads, hd)
    q = q_tensor_core(qkv[:, :q_dim].view(T, n_heads, hd), hd)
    r, where = _ratio(got, ref_prefill(q, c.kt, c.vt, p0, math.log(2)), visible_vmax(c.vt, p0, T, n_heads // n_kv), TOL_TC)
    assert r <= 1.0, f"err = {r:.3g} x bound at {where}"


@pytest.mark.gpu
@pytest.mark.parametrize("cache", CACHES)
def test_attn_prefill_deterministic(cache):
    n_heads, n_kv, hd, T, p0, seq = 32, 8, 128, 192, 192, 500
    qkv, c = _inputs(cache, n_heads, n_kv, hd, T, p0, seq)
    a = _tc(qkv, c, T, p0, n_heads, n_kv, hd, seq)
    b = _tc(qkv, c, T, p0, n_heads, n_kv, hd, seq)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.gpu
def test_attn_prefill_return_codes():
    """Shapes the kernel does not cover return 1 (the engine then runs the fallback); a chunk past the cache or a q80 call with one
    scale plane returns -1. None of them launches: the output keeps its sentinel."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    qkv = torch.zeros(1 << 20, device="cuda").data_ptr()
    kv = torch.zeros(1 << 20, dtype=torch.bfloat16, device="cuda")
    sc = torch.zeros(1 << 16, dtype=torch.float16, device="cuda")
    out = torch.full((1 << 20,), SENTINEL, dtype=torch.int16, device="cuda")
    k, v, s, o = kv.data_ptr(), kv[1 << 19:].data_ptr(), sc.data_ptr(), out.data_ptr()
    #          what                  rc  T   p0 nHeads nKv  hd  seqLen
    for what, want, T, p0, n_heads, n_kv, hd, seq in [("hd 96", 1, 4, 0, 4, 1, 96, 8), ("kvMul 256", 1, 2, 0, 256, 1, 64, 8),
                                                      ("nHeads % nKvHeads", 1, 2, 0, 12, 5, 64, 8), ("T 0", 1, 0, 0, 32, 8, 128, 8),
                                                      ("p0 + T > seqLen", -1, 4, 5, 32, 8, 128, 8)]:
        q_dim = n_heads * hd
        stride = q_dim + 2 * n_kv * hd
        assert lib.dl_attn_prefill_tc(qkv, stride, T, p0, n_heads, n_kv, hd, seq, k, v, o, q_dim, cl.stream_ptr()) == want, what
        assert lib.dl_attn_prefill_tc_q80(qkv, stride, T, p0, n_heads, n_kv, hd, seq, k, v, s, s, o, q_dim, cl.stream_ptr()) == want, what
    for ks, vs in ((s, None), (None, s)):
        rc = lib.dl_attn_prefill_tc_q80(qkv, 32 * 128 + 2 * 8 * 128, 4, 0, 32, 8, 128, 8, k, v, ks, vs, o, 32 * 128, cl.stream_ptr())
        assert rc == -1, ("one q80 scale plane", rc)
    torch.cuda.synchronize()
    assert (out == SENTINEL).all(), "a refused call launched the kernel"
