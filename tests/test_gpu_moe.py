"""Mixture-of-experts kernels against float64 references at Qwen3-30B-A3B expert shapes (128 experts, 8 active, dim 2048,
expert hidden size 768).

Kernels under test, through their stand-alone entry points:
* moeRouterKernel (decode_ops.cu): rmsnorm + f32 gate GEMV + top-k + softmax over the chosen logits, last CTA of a token selects.
* gemmQ40TcGrouped (grouped mode of gemmQ40TcTmaKernel, gemm_q40_tc.cu) with the GEPI_STORE_F32 and GEPI_SWIGLU_BF16 epilogues.
* moePrefillFfn (moe_prefill.cu): router, sort, gather, both grouped GEMMs, combine; one rank.
* The decode expert GEMVs (gemvQ40TmaKernel with moeCtasPerSlot, EPI_SWIGLU and EPI_MOE_DOWN), launched as the engine does.

The weights are random raw q40 blocks (uniform nibbles, f16 scales of about 1/(4 sqrt(n))). Every reference is computed in
float64 over exactly the values the kernel multiplies:
* tensor-core path: weights rn_bf16(rn_bf16(f16 scale) * (q - 8)) as the dequant warps build them, activations the bf16 rows the
  kernel reads (for the FFN, the kernel's own rmsnorm output, itself checked against float64), h rounded to bf16 after SwiGLU;
* decode path: q80-rounded activations (both stages) times the exact dequantised weights; stage 2 starts from the kernel's h;
* the FFN references take the routing the kernel used (ids and weights read back), so a near-tie in f32 cannot fail them.

Tolerances, derived from what is left after the shared roundings (S = sum |a * w| over the dot product of an output):
* f32 accumulation: 2^-18 * S, with S taken over |w| + 8 |scale| on the decode path (the GEMV multiplies unsigned nibbles and
  subtracts 8 * scale * sum(q) afterwards). At K = 2048 the tensor cores round the f32 accumulator once per k16 step, 128 times,
  each time by at most one ulp of a running sum that is at most S. Those roundings of random data add like a random walk
  (about sqrt(128) = 11 ulps); 2^-18 * S is 64 ulps. The GEMV rounds fewer times (per-block products, then ~40 sums).
* SiLU with __expf and fast division: 2^-19 relative.
* Roundings that both sides do, but from inputs that differ slightly: bf16(h) and the q80 grid (q = rint(x / d), d = f16(amax / 127)).
  The reference does not guess which way such a value went: it rounds both ends of the interval the kernel's input lies in. Where
  they agree the kernel's value must be that exact value; where they differ the bound gains the distance between them. The input
  interval is the f32 bound above for h; 2^-18 relative for the rmsnorm'd activations (fast rsqrt, f32 sum of squares, reciprocal
  and division approximations); 2^-20 relative for the kernel's h (reciprocal and division only).
* Routing weights: 2^-18 absolute (__expf of k logits, fast division).
* The residual add and the slot / pair sums in f32: 2^-22 of the magnitudes added.
A bound on one output therefore scales with S of that output. On an H100 80GB HBM3 (700 W) the bounds are at most 4.4e-5 of
max|ref| for the grouped GEMM, 4.3e-5 for the router logits and 1.1e-4 for the decode Δx. For the prefill Δx they reach 7e-3:
at the 30B shapes about one h element in seven can round to either bf16 neighbour, and each such element adds a bf16 ulp of h
times |w2|. All of these are below the 2 % of max|ref| that the dense GEMM tests use. The largest error is 0.12 of its bound for the
grouped GEMM, 0.54 for the prefill Δx, 0.05 for the router and 0.011 for the decode Δx. It is 0.81 for the sum of two
expert-parallel halves against the full run, whose bound covers f32 reordering only.
These changes to the reference each fail the tests named: tokens 64 and above of every group dropped (grouped GEMM and prefill
FFN), the f16 scale instead of its bf16 rounding (grouped GEMM at K = 2048), gate and up rows swapped (every SwiGLU check),
routing weights left unnormalised (router), and no q80 rounding of the kernel's h in decode stage 2 (decode FFN at 2048/768/128/8).
"""
import math

import pytest
import torch

from q40_ref import Experts, assert_bracketed, assert_within, bf16_bracket, f64_to_bf16, q80_ref, swiglu_ref
from q40_ref import gen as _gen, seed_of as _seed

pytestmark = pytest.mark.gpu

SILU = 0
EPS = 1e-6
C_ACC = 2.0 ** -18     # f32 accumulation, per unit of S
C_SUM = 2.0 ** -22     # residual add, slot / pair sums
REL_NORM = 2.0 ** -18  # kernel's rmsnorm'd f32 activations vs float64, relative
REL_H = 2.0 ** -20     # q80 of the kernel's own h: reciprocal and division only
TOL_W = 2.0 ** -18     # routing weights, absolute

SHAPE_30B = (2048, 768, 128, 8)
SHAPE_TINY = (256, 256, 8, 2)


def _cl():
    from distributed_llama_b200.ops import cuda_lib as cl
    return cl


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _i32(t):
    return t.to(torch.int32).contiguous().cuda()


# ---- float64 reference helpers ---------------------------------------------------------------------------------------
def rms_ref(x, w):
    x = x.double()
    return w.double() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS))


_EXPERTS = {}


def experts(E, rows, n, seed=0):
    key = (E, rows, n, seed)
    if key not in _EXPERTS:
        _EXPERTS[key] = Experts(E, rows, n, seed)
    return _EXPERTS[key]


def ffn_weights(dim, ff, E):
    """w13 [E][2 ff][dim] (gate rows even, up rows odd) and w2 [E][dim][ff]."""
    return experts(E, 2 * ff, dim, 1), experts(E, dim, ff, 2)


# ---- router ------------------------------------------------------------------------------------------------------------
def router_call(x, norm, gate, k, counter):
    cl = _cl()
    T, dim = x.shape
    E = gate.shape[0]
    logits = torch.full((T, E), float("nan"), device="cuda")
    ids = torch.full((T, k), -1, dtype=torch.int32, device="cuda")
    wts = torch.full((T, k), float("nan"), device="cuda")
    cl.check(cl.lib().dl_moe_router(x.data_ptr(), norm.data_ptr(), gate.data_ptr(), EPS, dim, E, k, logits.data_ptr(),
                                    counter.data_ptr(), ids.data_ptr(), wts.data_ptr(), T, cl.stream_ptr()), "moe_router")
    torch.cuda.synchronize()
    return logits, ids, wts


def router_check(x, norm, gate, k, logits, ids, wts, what):
    y = rms_ref(x, norm)
    g = gate.double()
    assert_within(logits, y @ g.T, C_ACC * (y.abs() @ g.abs().T), f"{what}: logits")
    # top-k of the kernel's own logits, descending, lowest index first among equal values
    want = torch.sort(logits, dim=1, descending=True, stable=True).indices[:, :k]
    assert torch.equal(ids.long(), want), f"{what}: chosen experts differ from the top-k of the logits"
    sel = torch.gather(logits.double(), 1, want)
    w_ref = torch.softmax(sel, dim=1)
    assert_within(wts, w_ref, torch.full_like(w_ref, TOL_W), f"{what}: routing weights")


ROUTER_SHAPES = [(256, 8, 2), (2048, 128, 8), (2048, 256, 8), (1024, 60, 4)]


def _router_inputs(dim, E, T, seed):
    g = _gen("router", dim, E, T, seed)
    x = torch.randn(T, dim, device="cuda", generator=g) * 2.0
    norm = 1.0 + 0.1 * torch.randn(dim, device="cuda", generator=g)
    gate = torch.randn(E, dim, device="cuda", generator=g) * (3.0 / math.sqrt(dim))
    return x, norm, gate


@pytest.mark.parametrize("T", [1, 37, 256])
@pytest.mark.parametrize("dim,E,k", ROUTER_SHAPES)
def test_router(dim, E, k, T):
    """Logits vs float64, ids = top-k of the kernel's logits, weights = softmax over the chosen logits; a second call on the same
    counter buffer is as correct as the first, and the counters are back at zero after each."""
    counter = torch.zeros(T + 16, dtype=torch.int32, device="cuda")
    counter[T:] = 0x7eadbeef
    for call in range(2):
        x, norm, gate = _router_inputs(dim, E, T, call)
        logits, ids, wts = router_call(x, norm, gate, k, counter)
        router_check(x, norm, gate, k, logits, ids, wts, f"router dim={dim} E={E} k={k} T={T} call {call}")
        assert (counter[:T] == 0).all(), "router counters not reset"
        assert (counter[T:] == 0x7eadbeef).all(), "router counters written past their end"


@pytest.mark.parametrize("dim,E,k", ROUTER_SHAPES)
def test_router_ties_pick_lowest_index(dim, E, k):
    """Experts 1, E/2 and E-1 (different CTAs) share one gate row aligned with every token: their logits are bitwise equal and the
    largest, so the first choices must be them in index order."""
    T = 37
    x, norm, gate = _router_inputs(dim, E, T, 9)
    c = torch.randn(dim, device="cuda", generator=_gen("tie", dim))
    c /= c.norm()
    x += 4.0 * math.sqrt(dim) * c / norm
    tied = [1, E // 2, E - 1]
    gate[tied] = 3.0 * c
    counter = torch.zeros(T, dtype=torch.int32, device="cuda")
    logits, ids, wts = router_call(x, norm, gate, k, counter)
    assert (logits[:, tied] == logits[:, 1:2]).all()
    router_check(x, norm, gate, k, logits, ids, wts, f"router ties dim={dim} E={E}")
    n = min(k, 3)
    assert (ids[:, :n] == torch.tensor(tied[:n], dtype=torch.int32, device="cuda")).all()


# ---- grouped tensor-core GEMM ------------------------------------------------------------------------------------------
EDGE_SIZES = [0, 1, 63, 64, 65, 127, 128, 129, 256]


def _group_sizes(pattern, G, max_tokens, seed):
    if pattern == "edges":
        sizes = [s for s in EDGE_SIZES if s <= max_tokens]
        return [sizes[i % len(sizes)] for i in range(G)]
    if pattern == "last":
        return [0] * (G - 1) + [max_tokens]
    g = torch.Generator().manual_seed(_seed("sizes", G, max_tokens, seed))
    return torch.randint(0, max_tokens + 1, (G,), generator=g).tolist()


def grouped_call(epi, w, G, grp_rows, act, counts, offsets, max_tokens, out):
    cl = _cl()
    cnt, off = _i32(counts), _i32(offsets)
    cl.check(cl.lib().dl_gemm_q40_tc_grouped(epi, w.qs.data_ptr(), w.scales.data_ptr(), G, grp_rows, act.shape[1], act.data_ptr(),
                                             act.stride(0), act.shape[0], max_tokens, cnt.data_ptr(), off.data_ptr(),
                                             out.data_ptr(), out.stride(0), _num_sms(), SILU, cl.stream_ptr()), "gemm_q40_tc_grouped")
    torch.cuda.synchronize()


@pytest.mark.parametrize("pattern,max_tokens", [("edges", 256), ("last", 256), ("random", 65)])
@pytest.mark.parametrize("G", [8, 128])
@pytest.mark.parametrize("grp_rows,n", [(1536, 2048), (2048, 768), (512, 256), (320, 256)])
def test_grouped_gemm(grp_rows, n, G, pattern, max_tokens):
    """Both epilogues of the grouped GEMM over the same groups. Groups are separated by a few unused activation rows; every row
    outside a group (and the tail TMA boxes read past the last one) is NaN. Outputs of group rows must be finite and within the
    bound; every other output row keeps its NaN fill."""
    cl = _cl()
    W = experts(G, grp_rows, n, 3)
    w = W.device()
    sizes = _group_sizes(pattern, G, max_tokens, 0)
    gaps = [(3 * g) % 5 for g in range(G)]
    offsets, r = [], 0
    for s, gp in zip(sizes, gaps):
        r += gp
        offsets.append(r)
        r += s
    rows_total = r + 64
    g = _gen("act", grp_rows, n, G, pattern)
    act = torch.full((rows_total, n), float("nan"), dtype=torch.bfloat16, device="cuda")
    inside = torch.zeros(rows_total, dtype=torch.bool, device="cuda")
    for o, s in zip(offsets, sizes):
        act[o:o + s] = torch.randn(s, n, device="cuda", generator=g).bfloat16()
        inside[o:o + s] = True
    counts = torch.tensor(sizes)
    offs = torch.tensor(offsets)
    out_f = torch.full((rows_total, grp_rows), float("nan"), device="cuda")
    out_h = torch.full((rows_total, grp_rows // 2), float("nan"), dtype=torch.bfloat16, device="cuda")
    grouped_call(cl.GEPI_STORE_F32, w, G, grp_rows, act, counts, offs, max_tokens, out_f)
    grouped_call(cl.GEPI_SWIGLU_BF16, w, G, grp_rows, act, counts, offs, max_tokens, out_h)
    what = f"grouped GEMM {grp_rows}x{n} G={G} {pattern} maxTokens={max_tokens}"
    assert torch.isnan(out_f[~inside]).all(), f"{what}: f32 output written outside the groups"
    assert torch.isnan(out_h[~inside].float()).all(), f"{what}: SwiGLU output written outside the groups"
    for e, (o, s) in enumerate(zip(offsets, sizes)):
        if s == 0:
            continue
        a = act[o:o + s].double()
        wt = W.w_tc(e)
        ref = a @ wt.T
        tol = C_ACC * (a.abs() @ wt.abs().T)
        assert_within(out_f[o:o + s], ref, tol, f"{what}: group {e} ({s} tokens) f32")
        h, eh = swiglu_ref(ref, tol)
        lo, hi = bf16_bracket(h, eh)
        assert_bracketed(out_h[o:o + s], lo, hi, f"{what}: group {e} ({s} tokens) SwiGLU")


# ---- prefill FFN -------------------------------------------------------------------------------------------------------
def planted_inputs(dim, E, routes, seed):
    """x [T][dim], norm and gate that route token t to the experts routes[t] (in that order) with a wide margin: gate row e is
    a scaled unit vector on coordinate e, and x[t] has large graded entries on the coordinates of its experts."""
    T, k = len(routes), len(routes[0])
    g = _gen("planted", dim, E, T, seed)
    x = torch.randn(T, dim, device="cuda", generator=g)
    x[:, :E] *= 0.1
    for t, r in enumerate(routes):
        x[t, torch.tensor(r, device="cuda")] = 6.0 + 0.5 * torch.arange(k, 0, -1, device="cuda", dtype=torch.float32)
    norm = 1.0 + 0.1 * torch.randn(dim, device="cuda", generator=g)
    norm[:E] = 1.0
    gate = torch.zeros(E, dim, device="cuda")
    gate[torch.arange(E), torch.arange(E)] = 0.5
    return x, norm, gate


def random_inputs(dim, E, T, seed):
    g = _gen("ffn", dim, E, T, seed)
    x = torch.randn(T, dim, device="cuda", generator=g)
    norm = 1.0 + 0.1 * torch.randn(dim, device="cuda", generator=g)
    gate = torch.randn(E, dim, device="cuda", generator=g) * (4.0 / math.sqrt(dim))
    return x, norm, gate


def prefill_call(x, norm, gate, W13, W2, ff, k, first=0, n_local=None):
    """moePrefillFfn on a copy of x; returns (new x, bf16 rmsnorm scratch, expert ids [T][k], weights [T][k])."""
    cl = _cl()
    T, dim = x.shape
    E = gate.shape[0]
    n_local = E - first if n_local is None else n_local
    w13, w2 = W13.device(first, n_local), W2.device(first, n_local)
    xo = x.clone()
    xn = torch.full((T, dim), float("nan"), dtype=torch.bfloat16, device="cuda")
    ids = torch.full((T, k), -1, dtype=torch.int32, device="cuda")
    wts = torch.full((T, k), float("nan"), device="cuda")
    cl.check(cl.lib().dl_moe_prefill_ffn(xo.data_ptr(), xn.data_ptr(), norm.data_ptr(), gate.data_ptr(), w13.qs.data_ptr(),
                                         w13.scales.data_ptr(), w2.qs.data_ptr(), w2.scales.data_ptr(), T, dim, ff, E, k, first, n_local,
                                         EPS, _num_sms(), SILU, ids.data_ptr(), wts.data_ptr(), cl.stream_ptr()), "moe_prefill_ffn")
    torch.cuda.synchronize()
    return xo, xn, ids, wts


def prefill_ref(xn, ids, wts, W13, W2, local=None):
    """Δx and its bound over the kernel's routing: per pair, bf16 activations times the tensor-core weights, h rounded to bf16.
    local = (first, count): only the pairs of those experts (one expert-parallel rank)."""
    T, dim = xn.shape
    dx = torch.zeros(T, dim, dtype=torch.float64, device="cuda")
    tol = torch.zeros_like(dx)
    mag = torch.zeros_like(dx)
    a_all = xn.double()
    for e in ids.unique().tolist():
        if local is not None and not (local[0] <= e < local[0] + local[1]):
            continue
        t, j = (ids == e).nonzero(as_tuple=True)
        a = a_all[t]
        w13, w2 = W13.w_tc(e), W2.w_tc(e)
        gu = a @ w13.T
        h, eh = swiglu_ref(gu, C_ACC * (a.abs() @ w13.abs().T))
        hb = f64_to_bf16(h)
        lo, hi = bf16_bracket(h, eh)
        y = hb @ w2.T
        ey = C_ACC * (hb.abs() @ w2.abs().T) + (hi - lo) @ w2.abs().T
        wt = wts[t, j].double()[:, None]
        dx.index_add_(0, t, wt * y)
        tol.index_add_(0, t, wt * ey)
        mag.index_add_(0, t, wt * y.abs())
    return dx, tol, mag


def prefill_check(x, norm, xo, xn, ids, wts, W13, W2, what, local=None):
    """xn vs float64 rmsnorm; Δx = xo - x vs the reference over the pairs of `local` experts (all when None)."""
    r = rms_ref(x, norm)
    lo, hi = bf16_bracket(r, REL_NORM * r.abs())
    assert_bracketed(xn, lo, hi, f"{what}: rmsnorm activations")
    dx, tol, mag = prefill_ref(xn, ids, wts, W13, W2, local)
    got = xo.double() - x.double()
    assert_within(got, dx, tol + C_SUM * (mag + xo.double().abs()), f"{what}: Δx")


@pytest.mark.parametrize("T", [9, 64, 65, 200, 256])
@pytest.mark.parametrize("dim,ff,E,k", [SHAPE_TINY, SHAPE_30B])
def test_prefill_ffn(dim, ff, E, k, T):
    """Random routing; a second run from the same x is bitwise equal."""
    W13, W2 = ffn_weights(dim, ff, E)
    x, norm, gate = random_inputs(dim, E, T, 0)
    xo, xn, ids, wts = prefill_call(x, norm, gate, W13, W2, ff, k)
    prefill_check(x, norm, xo, xn, ids, wts, W13, W2, f"prefill FFN {dim}/{ff}/{E}/{k} T={T}")
    xo2, _, ids2, wts2 = prefill_call(x, norm, gate, W13, W2, ff, k)
    assert torch.equal(xo, xo2) and torch.equal(ids, ids2) and torch.equal(wts, wts2), "two runs differ"


PLANTED_SIZES = {0: 256, 17: 256, 40: 256, 64: 256, 90: 256, 101: 256, 127: 256, 3: 65, 70: 64, 126: 63, 63: 1, 100: 63}


def planted_routes_30b():
    """256 tokens x 8 experts: seven experts get every token, the eighth choice gives groups of 65, 64, 63, 63 and 1 tokens."""
    eighth = [3] * 65 + [70] * 64 + [126] * 63 + [63] + [100] * 63
    every = [0, 17, 40, 64, 90, 101, 127]
    # graded order differs per token so that every slot position sees several experts
    return [every[t % 7:] + every[:t % 7] + [eighth[t]] for t in range(256)]


def test_prefill_ffn_planted_routing():
    """The 30B shape at T = 256 with the routing fixed by the inputs: one group per size that matters (256, 65, 64, 63, 1) and
    116 empty experts. The readback routing must have exactly these group sizes."""
    dim, ff, E, k = SHAPE_30B
    W13, W2 = ffn_weights(dim, ff, E)
    routes = planted_routes_30b()
    x, norm, gate = planted_inputs(dim, E, routes, 0)
    xo, xn, ids, wts = prefill_call(x, norm, gate, W13, W2, ff, k)
    assert torch.equal(ids.cpu(), torch.tensor(routes, dtype=torch.int32)), "planted routing not taken"
    sizes = torch.bincount(ids.flatten().long(), minlength=E).tolist()
    assert {e: s for e, s in enumerate(sizes) if s} == PLANTED_SIZES
    prefill_check(x, norm, xo, xn, ids, wts, W13, W2, "prefill FFN planted")
    xo2 = prefill_call(x, norm, gate, W13, W2, ff, k)[0]
    assert torch.equal(xo, xo2), "two runs differ"


def ep_routes(E, k, T, seed):
    """Distinct experts per token; the first 10 tokens use only experts of the lower half, the next 10 only the upper half."""
    g = torch.Generator().manual_seed(_seed("ep", E, k, T, seed))
    h = E // 2
    routes = []
    for t in range(T):
        lo, n = (0, h) if t < 10 else (h, h) if t < 20 else (0, E)
        routes.append((lo + torch.randperm(n, generator=g)[:k]).tolist())
    return routes


@pytest.mark.parametrize("dim,ff,E,k", [SHAPE_TINY, SHAPE_30B])
def test_prefill_ffn_expert_parallel(dim, ff, E, k):
    """Two expert-parallel halves on one GPU, each with only its experts' weights and its own copy of x: their Δx sum to the full
    run's within an f32 reordering bound, each half is correct on its own, and a token with no local expert keeps x bitwise."""
    T = 40
    W13, W2 = ffn_weights(dim, ff, E)
    routes = ep_routes(E, k, T, 0)
    x, norm, gate = planted_inputs(dim, E, routes, 1)
    full, _, ids, _ = prefill_call(x, norm, gate, W13, W2, ff, k)
    assert torch.equal(ids.cpu(), torch.tensor(routes, dtype=torch.int32)), "planted routing not taken"
    h = E // 2
    parts = []
    for first in (0, h):
        xo, xn, ids_p, wts_p = prefill_call(x, norm, gate, W13, W2, ff, k, first, h)
        assert torch.equal(ids_p, ids)
        prefill_check(x, norm, xo, xn, ids_p, wts_p, W13, W2, f"prefill FFN EP [{first}, {first + h})", local=(first, h))
        none_local = slice(10, 20) if first == 0 else slice(0, 10)
        assert torch.equal(xo[none_local], x[none_local]), "a token without local experts changed"
        parts.append(xo.double() - x.double())
    dfull = full.double() - x.double()
    bound = 2.0 ** -21 * (parts[0].abs() + parts[1].abs() + x.double().abs())
    assert_within(parts[0] + parts[1], dfull, bound, "prefill FFN EP: halves vs full")


def test_prefill_scratch_grows_with_token_count():
    """E = 128, k = 8, T = 32 followed by E = 8, k = 2, T = 128: the second call has fewer pairs but more tokens than the first,
    so the router's per-token scratch must grow with it."""
    for (dim, ff, E, k), T in ((SHAPE_30B, 32), (SHAPE_TINY, 128)):
        W13, W2 = ffn_weights(dim, ff, E)
        x, norm, gate = random_inputs(dim, E, T, 5)
        xo, xn, ids, wts = prefill_call(x, norm, gate, W13, W2, ff, k)
        counter = torch.zeros(T, dtype=torch.int32, device="cuda")
        _, ids_r, wts_r = router_call(x, norm, gate, k, counter)
        assert torch.equal(ids, ids_r) and torch.equal(wts, wts_r), f"T={T}: prefill routing differs from the router's"
        prefill_check(x, norm, xo, xn, ids, wts, W13, W2, f"scratch growth E={E} k={k} T={T}")


# ---- decode FFN --------------------------------------------------------------------------------------------------------
class DecodeBufs:
    def __init__(self, dim, ff, E, k, num_sms):
        z = dict(device="cuda")
        self.logits = torch.full((E,), float("nan"), **z)
        self.counter = torch.zeros(1 + 16, dtype=torch.int32, **z)
        self.ids = torch.full((k,), -1, dtype=torch.int32, **z)
        self.wts = torch.full((k,), float("nan"), **z)
        self.h = torch.full((k, ff), float("nan"), **z)
        self.scratch = torch.full((k, dim), float("nan"), **z)
        self.n_ctr = max(1, num_sms // k)
        self.counters = torch.zeros(self.n_ctr + 16, dtype=torch.int32, **z)
        self.counters[self.n_ctr:] = 0x7eadbeef
        self.counter[1:] = 0x7eadbeef

    def check(self, what):
        assert (self.counter[:1] == 0).all() and (self.counter[1:] == 0x7eadbeef).all(), f"{what}: router counter"
        assert (self.counters[:self.n_ctr] == 0).all(), f"{what}: slot counters not reset"
        assert (self.counters[self.n_ctr:] == 0x7eadbeef).all(), f"{what}: slot counters written past their end"


def decode_call(x, norm, gate, W13, W2, ff, k, num_sms, bufs, first=0, n_local=None):
    """One token; returns (x + weighted expert sum, h [k][ff], ids, weights)."""
    cl = _cl()
    dim = x.shape[0]
    E = gate.shape[0]
    n_local = E - first if n_local is None else n_local
    w13, w2 = W13.device(first, n_local), W2.device(first, n_local)
    out = x.clone()
    cl.check(cl.lib().dl_moe_decode_ffn(x.data_ptr(), out.data_ptr(), norm.data_ptr(), gate.data_ptr(), w13.qs.data_ptr(), w13.scales.data_ptr(),
                                        w2.qs.data_ptr(), w2.scales.data_ptr(), dim, ff, E, k, first, n_local, EPS, bufs.logits.data_ptr(),
                                        bufs.counter.data_ptr(), bufs.ids.data_ptr(), bufs.wts.data_ptr(), bufs.h.data_ptr(),
                                        bufs.scratch.data_ptr(), bufs.counters.data_ptr(), num_sms, SILU, cl.stream_ptr()), "moe_decode_ffn")
    torch.cuda.synchronize()
    return out, bufs.h.clone(), bufs.ids.clone(), bufs.wts.clone()


def decode_check(x, norm, out, h, ids, wts, W13, W2, what, local=None):
    """h per slot vs float64 from the q80 activations; Δx vs float64 from the kernel's own h. Slots whose expert is not local
    (expert parallelism) must give h = 0 and no contribution."""
    a1, amb1 = q80_ref(rms_ref(x, norm)[None], REL_NORM)
    dx = torch.zeros_like(x, dtype=torch.float64)
    tol = torch.zeros_like(dx)
    mag = torch.zeros_like(dx)
    for j, e in enumerate(ids.tolist()):
        if local is not None and not (local[0] <= e < local[0] + local[1]):
            assert (h[j] == 0).all(), f"{what}: slot {j} (expert {e}, not local) wrote h"
            continue
        w13, s13 = W13.w_exact(e)
        gu = (a1 @ w13.T)[0]
        e_gu = (C_ACC * (a1.abs() @ s13.T) + amb1 @ w13.abs().T)[0]
        h_ref, eh = swiglu_ref(gu, e_gu)
        assert_within(h[j], h_ref, eh, f"{what}: h of slot {j} (expert {e})")
        a2, amb2 = q80_ref(h[j].double()[None], REL_H)
        w2, s2 = W2.w_exact(e)
        y = (a2 @ w2.T)[0]
        ey = (C_ACC * (a2.abs() @ s2.T) + amb2 @ w2.abs().T)[0]
        wt = wts[j].double()
        dx += wt * y
        tol += wt * ey
        mag += wt * y.abs()
    got = out.double() - x.double()
    assert_within(got, dx, tol + C_SUM * (mag + out.double().abs()), f"{what}: Δx")


DECODE_SHAPES = [SHAPE_TINY, SHAPE_30B, (2048, 384, 128, 8)]


@pytest.mark.parametrize("sms", ["device", 17])
@pytest.mark.parametrize("dim,ff,E,k", DECODE_SHAPES)
def test_decode_ffn(dim, ff, E, k, sms):
    """Four tokens through the same buffers (self-resetting counters); each run twice, bitwise equal. sms = 17 gives 2 CTAs per
    routing slot at k = 8 and 8 at k = 2 instead of the engine's 16 / 66."""
    num_sms = _num_sms() if sms == "device" else sms
    W13, W2 = ffn_weights(dim, ff, E)
    bufs = DecodeBufs(dim, ff, E, k, num_sms)
    x, norm, gate = random_inputs(dim, E, 4, 7)
    for t in range(4):
        what = f"decode FFN {dim}/{ff}/{E}/{k} sms={num_sms} token {t}"
        out, h, ids, wts = decode_call(x[t], norm, gate, W13, W2, ff, k, num_sms, bufs)
        bufs.check(what)
        decode_check(x[t], norm, out, h, ids, wts, W13, W2, what)
        out2, h2, ids2, wts2 = decode_call(x[t], norm, gate, W13, W2, ff, k, num_sms, bufs)
        assert torch.equal(out, out2) and torch.equal(h, h2) and torch.equal(ids, ids2) and torch.equal(wts, wts2), f"{what}: two runs differ"


@pytest.mark.parametrize("dim,ff,E,k", [SHAPE_TINY, SHAPE_30B])
def test_decode_ffn_expert_parallel(dim, ff, E, k):
    """Halves [0, E/2) and [E/2, E) with their own weights: the Δx sum to the full run's within an f32 reordering bound; a token
    routed only to lower-half experts leaves x bitwise unchanged on the upper half."""
    num_sms = _num_sms()
    W13, W2 = ffn_weights(dim, ff, E)
    routes = ep_routes(E, k, 21, 1)
    x, norm, gate = planted_inputs(dim, E, routes, 2)
    h_ = E // 2
    for t in (0, 20):                      # token 0: lower-half experts only; token 20: mixed
        bufs = DecodeBufs(dim, ff, E, k, num_sms)
        full, _, ids, _ = decode_call(x[t], norm, gate, W13, W2, ff, k, num_sms, bufs)
        assert ids.tolist() == routes[t], "planted routing not taken"
        parts = []
        for first in (0, h_):
            out, h, ids_p, wts_p = decode_call(x[t], norm, gate, W13, W2, ff, k, num_sms, bufs, first, h_)
            bufs.check(f"decode EP token {t} [{first}, {first + h_})")
            decode_check(x[t], norm, out, h, ids_p, wts_p, W13, W2, f"decode FFN EP token {t} [{first}, {first + h_})", local=(first, h_))
            if t == 0 and first == h_:
                assert torch.equal(out, x[t]), "a token without local experts changed"
            parts.append(out.double() - x[t].double())
        bound = 2.0 ** -21 * (parts[0].abs() + parts[1].abs() + x[t].double().abs())
        assert_within(parts[0] + parts[1], full.double() - x[t].double(), bound, f"decode FFN EP token {t}: halves vs full")


# ---- engine --------------------------------------------------------------------------------------------------------------
def test_engine_moe_prefill_one_chunk(tmp_models):
    """tiny-qwen3-moe: a 250-token prompt as one tensor-core chunk (both layers reuse the MoE scratch) against the oracle and
    against the GEMV path of the same engine, at the tolerance of the other engine tests."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    from distributed_llama_b200.runtime import Engine
    mf = ModelFile(tmp_models["tiny-qwen3-moe"][0])
    toks = [(11 * i + 5) % 500 + 1 for i in range(250)]
    ref = OracleModel(mf, act_quant="q80", device="cuda").forward(toks, 0)[-1]
    eng = Engine(load_device_weights(mf), max_prefill=256)
    lg = eng.prefill(toks, 0).clone()
    assert (lg - ref).abs().max().item() < 0.12
    eng_b = Engine(load_device_weights(mf), max_prefill=256)
    eng_b.use_tc_prefill = False
    lg_b = eng_b.prefill(toks, 0)
    assert (lg - lg_b).abs().max().item() < 0.12
