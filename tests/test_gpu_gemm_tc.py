"""Dense prefill GEMM (gemm_q40_tc.cu: gemmQ40TcKernel "ldg", gemmQ40TcTmaKernel "tma") and rmsNormBf16Kernel against float64.

Every case asserts the path it runs through dl_gemm_q40_tc_plan (kernel, split-K count, cluster or global-scratch reduce), so a
change of the dispatch heuristic fails here instead of silently moving a case off its path. The paths are steered with num_sms,
DL_GEMM_SPLITK and DL_GEMM_CLUSTER; num_sms never exceeds the device's SM count (the global-scratch reduce needs all splits of an
item co-resident), and the forced-path shapes reach their plans at 48 SMs, so they run the same way on every H100.

Reference: float64 over exactly what the tensor cores multiply: the bf16 activation rows, and weights
rn_bf16(rn_bf16(f16 scale) * (q - 8)) as the dequant warps build them (q40_ref.w_tc_of). Bounds, per output element, with
S = sum_k |a_k w_k| of that output:
* f32 accumulation: 2^-18 * S. The tensor cores round the f32 accumulator once per k16 step (K / 16 times), each time by at most
  an ulp (2^-23 relative) of a running sum that is at most S. Random-sign roundings add like a random walk: at K = 28672 that is
  about sqrt(1792) = 42 half-ulps of S, 2^-18.6 * S; 2^-18 * S is 64 ulps.
* Split-K partial sums, added in f32 in rank order from 0, and the residual add: 2^-22 of the magnitudes added (at most four
  roundings of sums no larger than S + |residual| + |result|).
* SwiGLU stores bf16: the reference rounds both ends of the interval the kernel's f32 value lies in (bf16_bracket); the
  kernel's value must lie between them.
* SiLU (__expf, fast division): 2^-19 relative. tanh-GELU (tanhf, f32 polynomial argument): 2^-20 * (|gelu(g)| + |g|); the
  absolute term covers the cancellation in 1 + tanh(u) for negative g. The bound on g and up carries through the derivatives
  |silu'| <= 1.1 and |gelu'| <= 1.13.
* rmsnorm: 2^-18 relative (f32 sum of squares over <= 45 additions, rsqrtf, two products), bracketed to bf16.

Exactness: with one-hot activation rows (token t has 1.0 at column k_t) out[t, f] must equal w_tc[f, k_t] exactly, whatever the
path: every other product is a signed zero and the split-K partials of the other ranges are zeros. That pins nibble order, the
SWIZZLE_128B chunk mapping, scale placement, row and token tiles and the K range of every split.

On an H100 80GB HBM3 (132 SMs, 700 W power limit) the largest error / bound of an f32 output is 0.26 on the register-prefetch
kernel, 0.30 on the TMA-staged one without a split, 0.12 / 0.11 with a 2-way cluster / global-scratch reduce, 0.079 with the 3-way
global one and 0.052 / 0.024 with a 4-way cluster / global one. The file runs in about 10 s there.
These changes to the kernel each fail the tests named: dequant offset 136 -> 135, the f16 scale multiplied in f32 and rounded once,
two nibble shifts swapped, split ks > 0 starting one raw chunk early (out = 2w) and the global reduce dropping the last split
(one-hot exactness); the cluster reduce skipping its peers' partials at tok = tEnd - 1 (one-hot, cluster paths); gate and up rows
swapped (every SwiGLU case, 7 away from the interval) and the residual read from token + 1 (24700 x the bound).
"""
import pytest
import torch

from q40_ref import Experts, assert_bracketed, assert_within, bf16_bracket, gen, q40_parts, w_tc_of

C_ACC = 2.0 ** -18
C_SUM = 2.0 ** -22
C_SILU = 2.0 ** -19
C_GELU = 2.0 ** -20
REL_NORM = 2.0 ** -18
SILU, GELU = 0, 1
NAN_F32 = 0x7FC0DEAD          # payload written around the outputs: must survive every call
NAN_BF16 = 0x7FD5

# gemm_q40_tc.cu GEPI_*
F32, RESID, SWIGLU = 0, 1, 2
EPILOGUES = {"f32": (F32, SILU), "residual": (RESID, SILU), "swiglu-silu": (SWIGLU, SILU), "swiglu-gelu": (SWIGLU, GELU)}

T_EDGES = [1, 16, 63, 64, 65, 127, 128, 129, 192, 255, 256]


def _ops():
    from distributed_llama_b200 import ops
    return ops


def _device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- production shapes: (d, n) of QKV, WO, W1|W3, W2 per model; plans at 132 SMs pinned from the dispatch code --------------
MODELS = {
    "llama-3.1-8b": {"qkv": (6144, 4096), "wo": (4096, 4096), "w13": (28672, 4096), "w2": (4096, 14336)},
    "qwen3-8b": {"qkv": (6144, 4096), "wo": (4096, 4096), "w13": (24576, 4096), "w2": (4096, 12288)},
    "qwen3-14b": {"qkv": (7168, 5120), "wo": (5120, 5120), "w13": (34816, 5120), "w2": (5120, 17408)},
    "qwen3-0.6b": {"qkv": (4096, 1024), "wo": (1024, 2048), "w13": (6144, 1024), "w2": (1024, 3072)},
    # also Llama-3.1-8B at 8-way tensor parallelism (one rank's slices)
    "llama-3.1-8b-slice8": {"qkv": (768, 4096), "wo": (4096, 512), "w13": (3584, 4096), "w2": (4096, 1792)},
    "qwen3-14b-tp8": {"qkv": (896, 5120), "wo": (5120, 640), "w13": (4352, 5120), "w2": (5120, 2176)},
    "llama-3.3-70b-tp8": {"qkv": (1280, 8192), "wo": (8192, 1024), "w13": (7168, 8192), "w2": (8192, 3584)},
}
MATRIX_EPI = {"qkv": F32, "wo": RESID, "w13": SWIGLU, "w2": RESID}     # enginePrefill on one GPU
PLAN_TS = [1, 16, 63, 64, 65, 128, 192, 256]
# (kernel, splitK, cluster) per T in PLAN_TS at 132 SMs; kernel 1 = ldg, 2 = tma. "n" no split, "c2"/"c4" cluster, "g3" global.
_P = {"n": (2, 1, 0), "c2": (2, 2, 1), "c4": (2, 4, 1), "g3": (2, 3, 0), "ldg": (1, 1, 0)}
PLAN_TABLE = {
    ("llama-3.1-8b", "qkv"): "n n n n n n n n", ("llama-3.1-8b", "wo"): "c4 c4 c4 c4 n n n n",
    ("llama-3.1-8b", "w13"): "n n n n n n n n", ("llama-3.1-8b", "w2"): "c4 c4 c4 c4 c2 c2 n n",
    ("qwen3-8b", "qkv"): "n n n n n n n n", ("qwen3-8b", "wo"): "c4 c4 c4 c4 n n n n",
    ("qwen3-8b", "w13"): "n n n n n n n n", ("qwen3-8b", "w2"): "c4 c4 c4 c4 c2 c2 n n",
    ("qwen3-14b", "qkv"): "n n n n n n n n", ("qwen3-14b", "wo"): "n n n n n n n n",
    ("qwen3-14b", "w13"): "n n n n n n n n", ("qwen3-14b", "w2"): "g3 g3 g3 g3 n n n n",
    ("qwen3-0.6b", "qkv"): "n n n n n n n n", ("qwen3-0.6b", "wo"): "n n n n n n n n",
    ("qwen3-0.6b", "w13"): "n n n n n n n n", ("qwen3-0.6b", "w2"): "n n n n n n n n",
    ("llama-3.1-8b-slice8", "qkv"): "c4 c4 c4 c4 c4 c4 c4 c4", ("llama-3.1-8b-slice8", "wo"): "n n n n n n n n",
    ("llama-3.1-8b-slice8", "w13"): "c4 c4 c4 c4 n n n n", ("llama-3.1-8b-slice8", "w2"): "n n n n n n n n",
    ("qwen3-14b-tp8", "qkv"): "c4 c4 c4 c4 c4 c4 c4 c4", ("qwen3-14b-tp8", "wo"): "ldg ldg ldg ldg ldg ldg ldg ldg",
    ("qwen3-14b-tp8", "w13"): "n n n n n n n n", ("qwen3-14b-tp8", "w2"): "ldg ldg ldg ldg ldg ldg ldg ldg",
    ("llama-3.3-70b-tp8", "qkv"): "c4 c4 c4 c4 c4 c4 c4 g3", ("llama-3.3-70b-tp8", "wo"): "n n n n n n n n",
    ("llama-3.3-70b-tp8", "w13"): "c2 c2 c2 c2 n n n n", ("llama-3.3-70b-tp8", "w2"): "n n n n n n n n",
}


def _pinned(model, mat, T):
    return _P[PLAN_TABLE[model, mat].split()[PLAN_TS.index(T)]]


def _path(plan):
    return (plan.kernel, plan.split_k, plan.cluster)


def test_plan_table_at_132_sms():
    """Production shapes at 132 SMs (H100 SXM): the plans the dispatch picked when this table was written, e.g. Llama-3.1-8B W2
    takes a 4-way cluster reduce at 64 tokens, a 2-way one at 128 and none at 192; Qwen3-14B W2 the 3-way global-scratch
    reduce at <= 64 tokens. The plan launches nothing, so this runs without a GPU."""
    ops = _ops()
    for (model, mat), row in PLAN_TABLE.items():
        d, n = MODELS[model][mat]
        for T in PLAN_TS:
            p = ops.gemm_q40_tc_plan(MATRIX_EPI[mat], d, n, T, num_sms=132)
            assert p.rc == 0 and p.grid <= 132, (model, mat, T, p)
            assert _path(p) == _pinned(model, mat, T), f"{model} {mat} T={T}: {p}"
            if p.kernel == 2:
                assert (p.stages, p.raw_stages, p.b_stages) == (8, 3, 4), p


def test_plan_switches(monkeypatch):
    """DL_GEMM_SPLITK lowers the split count, DL_GEMM_CLUSTER=0 moves 2- and 4-way splits to the global scratch; both are read by
    the plan exactly as by the launch."""
    ops = _ops()
    base = dict(epi=F32, d=FD, n=FN, T=256)
    for sk, cl, want in [(None, None, (2, 4, 1)), (None, "0", (2, 4, 0)), ("3", None, (2, 3, 0)), ("2", None, (2, 2, 1)),
                         ("2", "0", (2, 2, 0)), ("1", None, (2, 1, 0)), ("9", None, (2, 4, 1))]:
        for k, v in (("DL_GEMM_SPLITK", sk), ("DL_GEMM_CLUSTER", cl)):
            if v is None:
                monkeypatch.delenv(k, raising=False)
            else:
                monkeypatch.setenv(k, v)
        p = ops.gemm_q40_tc_plan(base["epi"], base["d"], base["n"], base["T"], num_sms=FSMS)
        assert _path(p) == want and p.grid == 12 * p.split_k, (sk, cl, p)


def test_w_tc_model_and_one_hot_rows():
    """CPU: the tensor-core weight model on hand-computed blocks (negative scale, nibble 8, both nibbles of a byte, a scale whose
    bf16 rounding matters) and the one-hot activation rows of the exactness test."""
    raw = torch.zeros(2, 18, dtype=torch.uint8)
    raw[0, :2] = torch.tensor([-0.5], dtype=torch.float16).view(torch.uint8)
    raw[0, 2:] = 0x88
    raw[0, 2] = 0x0F          # element 0: q = 15, element 16: q = 0
    raw[0, 3] = 0x81          # element 1: q = 1,  element 17: q = 8
    raw[1, :2] = torch.tensor([0.1], dtype=torch.float16).view(torch.uint8)   # f16 0.0999755859375 -> bf16 0.10009765625
    raw[1, 2:] = 0x88
    raw[1, 2] = 0xC9          # element 0: q = 9, element 16: q = 12
    raw[1, 17] = 0x1F         # element 15: q = 15, element 31: q = 1
    sc, q = q40_parts(raw, 1, 64)
    w = w_tc_of(sc, q)[0]
    want = torch.zeros(64, dtype=torch.float64)
    want[0], want[16], want[1], want[17] = -3.5, 4.0, 3.5, 0.0
    want[32], want[48], want[47], want[63] = 0.10009765625, 0.400390625, 0.69921875, -0.69921875
    assert torch.equal(w, want), (w[w != want], want[w != want])
    assert w[17].item() == 0.0 and (w[2:16] == 0).all() and (w[33:47] == 0).all()
    for n in (256, 4352):
        cols = torch.zeros(n, dtype=torch.int64)
        for launch in range(n // 256):
            a, k = one_hot_rows(n, launch, "cpu")
            assert a.dtype == torch.bfloat16 and (a.float().sum(1) == 1).all() and (a.float().amax(1) == 1).all()
            assert torch.equal(a.float().argmax(1), k) and k.unique().numel() == 256
            cols[k] += 1
        assert (cols == 1).all(), "the launches must cover every column exactly once"


def one_hot_rows(n, launch, device="cuda"):
    """256 one-hot bf16 rows covering columns [256 launch, 256 launch + 256) in a token order that differs per launch."""
    t = torch.arange(256)
    k = 256 * launch + (37 * t + 11 * launch) % 256
    a = torch.zeros(256, n, dtype=torch.bfloat16)
    a[t, k] = 1.0
    return a.to(device), k.to(device)


# ---- GPU cases -----------------------------------------------------------------------------------------------------------
def _run(w, act, epi, out, *, num_sms, variant="auto", act_fn=SILU):
    _ops().gemm_q40_tc(w, act, epi=epi, out=out, num_sms=num_sms, variant=variant, act_fn=act_fn)
    torch.cuda.synchronize()
    return out


def _glu_ref(gu, e_gu, act_fn):
    """h = act(gate) * up from interleaved rows (gate even, up odd) and the bound on the kernel's f32 h."""
    g, u, eg, eu = gu[..., 0::2], gu[..., 1::2], e_gu[..., 0::2], e_gu[..., 1::2]
    if act_fn == SILU:
        s = g / (1.0 + torch.exp(-g))
        d, e_act = 1.1, C_SILU * s.abs()
    else:
        s = 0.5 * g * (1.0 + torch.tanh(0.7978845608028654 * g * (1.0 + 0.044715 * g * g)))
        d, e_act = 1.13, C_GELU * (s.abs() + g.abs())
    h = s * u
    return h, d * eg * u.abs() + s.abs() * eu + d * eg * eu + e_act * u.abs() + 2.0 ** -24 * h.abs()


def check_output(epi, act_fn, got, ref, S, x0, what):
    """got: the kernel's output rows; ref / S: float64 a @ w^T and |a| @ |w|^T of the same rows; x0: residual (RESID).
    Returns the largest error / bound of the f32 outputs (None for the bracketed bf16 ones)."""
    tol = C_ACC * S + C_SUM * S
    if epi == F32:
        return assert_within(got, ref, tol, what)
    if epi == RESID:
        r = x0.double() + ref
        return assert_within(got, r, tol + C_SUM * (x0.double().abs() + r.abs()), what)
    lo, hi = bf16_bracket(*_glu_ref(ref, tol, act_fn))
    assert_bracketed(got, lo, hi, what)
    return None


def _out_cols(epi, d):
    return d // 2 if epi == SWIGLU else d


def _out_dtype(epi):
    return torch.float32 if epi in (F32, RESID) else torch.bfloat16


class Case:
    """Random q40 matrix [d][n], 256 random bf16 activation rows, a residual; float64 reference over all 256 rows (a token's
    output does not depend on T)."""

    def __init__(self, d, n, seed=0):
        W = Experts(1, d, n, seed)
        self.d, self.n, self.w = d, n, W.device()
        g = gen("act", d, n, seed)
        self.act = torch.randn(256, n, device="cuda", generator=g).bfloat16()
        self.x0 = torch.randn(256, d, device="cuda", generator=g)
        wt = W.w_tc()
        self.ref = self.act.double() @ wt.T
        self.S = (self.act.float().abs() @ wt.float().abs().T).double()     # the scale of a bound: f32 is plenty
        del wt

    def out_buf(self, epi, T):
        if epi == RESID:
            return self.x0[:T].clone()
        return torch.full((T, _out_cols(epi, self.d)), float("nan"), dtype=_out_dtype(epi), device="cuda")

    def run(self, epi, T, *, num_sms, variant="auto", act_fn=SILU):
        return _run(self.w, self.act[:T], epi, self.out_buf(epi, T), num_sms=num_sms, variant=variant, act_fn=act_fn)

    def check(self, epi, act_fn, got, T, what):
        return check_output(epi, act_fn, got, self.ref[:T], self.S[:T], self.x0[:T], what)


_CASES = {}


def case(d, n, seed=0):
    if (d, n, seed) not in _CASES:
        _CASES.clear()          # production shapes are large: keep one at a time
        _CASES[d, n, seed] = Case(d, n, seed)
    return _CASES[d, n, seed]


RATIOS = {}    # largest error / bound seen per path (kernel, splitK, cluster) in this process, for reports


def _note(path, r):
    if r is not None:
        RATIOS[path] = max(RATIOS.get(path, 0.0), r)


@pytest.mark.gpu
@pytest.mark.parametrize("model,mat", list(PLAN_TABLE))
def test_production_shapes(model, mat):
    """QKV, WO, W1|W3, W2 with the engine's epilogue at T in PLAN_TS on all of the device's SMs; on a 132-SM H100 each launch
    must take the pinned plan."""
    ops = _ops()
    d, n = MODELS[model][mat]
    epi = MATRIX_EPI[mat]
    sms = _device_sms()
    c = case(d, n)
    for T in PLAN_TS:
        p = ops.gemm_q40_tc_plan(epi, d, n, T, num_sms=sms)
        if sms == 132:
            assert _path(p) == _pinned(model, mat, T), (model, mat, T, p)
        r = c.check(epi, SILU, c.run(epi, T, num_sms=sms), T, f"{model} {mat} {d}x{n} T={T} plan {_path(p)}")
        _note(_path(p), r)


# Forced paths: one shape that reaches a 4-way split at every T with 48 SMs (3 row tiles, the last one half full; 17 raw K chunks
# so that no split count divides K evenly), steered down to 3, 2 and 1 splits and between the two reduce schemes.
FD, FN, FSMS = 320, 4352, 48
PATHS = {   # name: (variant, DL_GEMM_SPLITK, DL_GEMM_CLUSTER, num_sms, expected (kernel, splitK, cluster))
    "ldg": ("ldg", None, None, FSMS, (1, 1, 0)),
    "tma-s1-c1": ("tma", "1", "1", FSMS, (2, 1, 0)),
    "tma-s1-c0": ("tma", "1", "0", FSMS, (2, 1, 0)),
    "cluster2": ("tma", "2", "1", FSMS, (2, 2, 1)),
    "global2": ("tma", "2", "0", FSMS, (2, 2, 0)),
    "global3-c1": ("tma", "3", "1", FSMS, (2, 3, 0)),
    "global3-c0": ("tma", "3", "0", FSMS, (2, 3, 0)),
    "cluster4": ("auto", None, None, FSMS, (2, 4, 1)),
    "global4": ("auto", None, "0", FSMS, (2, 4, 0)),
    "tma-3sms": ("tma", None, None, 3, (2, 1, 0)),      # 12 to 15 work items per CTA: every ring wraps many times
    "ldg-7sms": ("ldg", None, None, 7, (1, 1, 0)),
}
EXACT_PATHS = ["ldg", "tma-s1-c1", "cluster2", "global2", "global3-c0", "cluster4", "global4"]


def _steer(monkeypatch, name):
    variant, sk, cl, sms, want = PATHS[name]
    for k, v in (("DL_GEMM_SPLITK", sk), ("DL_GEMM_CLUSTER", cl)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    assert sms <= _device_sms()
    return variant, sms, want


def _assert_plan(epi, d, n, T, sms, variant, want, act_stride=None):
    p = _ops().gemm_q40_tc_plan(epi, d, n, T, act_stride=act_stride, num_sms=sms, variant=variant)
    assert p.rc == 0 and _path(p) == want, f"{d}x{n} T={T} sms={sms} {variant}: plan {p}, expected {want}"


@pytest.mark.gpu
@pytest.mark.parametrize("path", EXACT_PATHS)
def test_one_hot_exact(path, monkeypatch):
    """One-hot rows: out[t, f] == w_tc[f, k_t] for every (f, k) of the matrix, 256 tokens per launch, on every kernel and split
    path."""
    variant, sms, want = _steer(monkeypatch, path)
    W = Experts(1, FD, FN, 11)
    w, wt = W.device(), W.w_tc().float()
    for launch in range(FN // 256):
        a, k = one_hot_rows(FN, launch)
        _assert_plan(F32, FD, FN, 256, sms, variant, want)
        out = _run(w, a, F32, torch.full((256, FD), float("nan"), device="cuda"), num_sms=sms, variant=variant)
        ref = wt[:, k].T
        bad = out != ref
        if bad.any():
            t, f = bad.nonzero()[0].tolist()
            raise AssertionError(f"{path} launch {launch}: {int(bad.sum())} outputs differ; token {t} (column {k[t].item()}) row {f}: "
                                 f"{out[t, f].item()!r} != w_tc {ref[t, f].item()!r}")


def _padded(act, T, n_pad):
    """act[:T] inside a NaN-filled buffer with 64 more rows and n_pad more columns (actStride = n + n_pad)."""
    n = act.shape[1]
    buf = torch.full((T + 64, n + n_pad), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:T, :n] = act[:T]
    return buf[:T, :n]


def _payload_out(epi, T, cols, inside=None):
    """[T + 3][cols + 40] filled with a NaN payload; the [T][cols] view starts one row and 8 columns in."""
    if _out_dtype(epi) == torch.float32:
        buf = torch.full((T + 3, cols + 40), NAN_F32, dtype=torch.int32, device="cuda").view(torch.float32)
    else:
        buf = torch.full((T + 3, cols + 40), NAN_BF16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    view = buf[1:T + 1, 8:8 + cols]
    if inside is not None:
        view.copy_(inside)
    return buf, view


def _payload_intact(buf, T, cols):
    ints = buf.view(torch.int32 if buf.dtype == torch.float32 else torch.int16)
    mask = torch.ones_like(ints, dtype=torch.bool)
    mask[1:T + 1, 8:8 + cols] = False
    want = NAN_F32 if buf.dtype == torch.float32 else NAN_BF16
    return bool((ints[mask] == want).all())


@pytest.mark.gpu
@pytest.mark.parametrize("epi_name", list(EPILOGUES))
@pytest.mark.parametrize("path", list(PATHS))
def test_forced_paths(path, epi_name, monkeypatch):
    """Every epilogue on every kernel / split path at the token-tile edges. Then, at T = 65 and 256: the same call with act a
    strided view (actStride = n + 72) inside NaN padding and out a strided view inside a NaN payload gives bitwise the same values
    and leaves the payload alone; three repeats are bitwise equal."""
    epi, act_fn = EPILOGUES[epi_name]
    variant, sms, want = _steer(monkeypatch, path)
    c = case(FD, FN)
    cols = _out_cols(epi, FD)
    for T in T_EDGES:
        _assert_plan(epi, FD, FN, T, sms, variant, want)
        got = c.run(epi, T, num_sms=sms, variant=variant, act_fn=act_fn)
        _note(want, c.check(epi, act_fn, got, T, f"{path} {epi_name} T={T}"))
        if T not in (65, 256):
            continue
        _assert_plan(epi, FD, FN, T, sms, variant, want, act_stride=FN + 72)
        buf, view = _payload_out(epi, T, cols, c.x0[:T] if epi == RESID else None)
        _run(c.w, _padded(c.act, T, 72), epi, view, num_sms=sms, variant=variant, act_fn=act_fn)
        assert torch.equal(view, got), f"{path} {epi_name} T={T}: strided / padded call differs from the plain one"
        assert _payload_intact(buf, T, cols), f"{path} {epi_name} T={T}: written outside [T, {cols}]"
        for _ in range(3):
            again = c.run(epi, T, num_sms=sms, variant=variant, act_fn=act_fn)
            assert torch.equal(again, got), f"{path} {epi_name} T={T}: repeat differs"


@pytest.mark.gpu
@pytest.mark.parametrize("epi_name", ["f32", "residual", "swiglu-gelu"])
def test_cross_path_identity(epi_name, monkeypatch):
    """ldg and tma without a split issue the same wgmma sequence on the same tiles; the cluster and global-scratch reduces add the
    same partials in the same order from 0. Each pair must agree bitwise."""
    epi, act_fn = EPILOGUES[epi_name]
    c = case(FD, FN)
    for T in (1, 65, 256):
        res = {}
        for path in ("ldg", "tma-s1-c1", "cluster2", "global2", "cluster4", "global4"):
            variant, sms, want = _steer(monkeypatch, path)
            _assert_plan(epi, FD, FN, T, sms, variant, want)
            res[path] = c.run(epi, T, num_sms=sms, variant=variant, act_fn=act_fn)
        for a, b in (("ldg", "tma-s1-c1"), ("cluster2", "global2"), ("cluster4", "global4")):
            assert torch.equal(res[a], res[b]), f"{epi_name} T={T}: {a} and {b} differ by up to {(res[a].double() - res[b].double()).abs().max().item():.3g}"


# Other shapes: TMA with d % 128 != 0 at a large d, the register-prefetch kernel with n % 256 != 0 (auto picks it), small grids.
SHAPES = [   # (d, n, variant, num_sms or 0 = device, expected kernel)
    (1000, 2048, "auto", 0, 2), (5184, 1024, "auto", 0, 2), (1000, 2176, "auto", 0, 1), (320, 960, "auto", 0, 1),
    (1000, 2048, "tma", 1, 2), (1000, 2048, "tma", 7, 2), (1000, 2176, "ldg", 3, 1), (5184, 1024, "ldg", 0, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("d,n,variant,sms,kernel", SHAPES)
def test_shapes(d, n, variant, sms, kernel):
    sms = sms or _device_sms()
    c = case(d, n, 1)
    for epi_name in ("f32", "residual", "swiglu-silu", "swiglu-gelu"):
        epi, act_fn = EPILOGUES[epi_name]
        for T in (1, 63, 65, 129, 200, 256):
            p = _ops().gemm_q40_tc_plan(epi, d, n, T, num_sms=sms, variant=variant)
            assert p.rc == 0 and p.kernel == kernel and p.split_k == 1, p
            got = c.run(epi, T, num_sms=sms, variant=variant, act_fn=act_fn)
            _note(_path(p), c.check(epi, act_fn, got, T, f"{d}x{n} {variant} sms={sms} {epi_name} T={T}"))


@pytest.mark.gpu
def test_split_scratch_reuse_and_growth(monkeypatch):
    """The global-scratch reduce's buffer and self-resetting counters across shapes: a 4-way split, a 3-way split of another
    shape (fewer row tiles, other token tiles), then a call that needs more scratch than both (grows the buffer in a fresh
    process), then the first again."""
    monkeypatch.setenv("DL_GEMM_CLUSTER", "0")
    seq = [(320, 4352, 256, 48, None, 4), (256, 4096, 128, 32, "3", 3), (896, 4096, 256, 112, None, 4), (320, 4352, 256, 48, None, 4)]
    for d, n, T, sms, sk, want in seq:
        if sms > _device_sms():
            pytest.skip(f"needs {sms} SMs")
        if sk is None:
            monkeypatch.delenv("DL_GEMM_SPLITK", raising=False)
        else:
            monkeypatch.setenv("DL_GEMM_SPLITK", sk)
        _assert_plan(RESID, d, n, T, sms, "auto", (2, want, 0))
        c = case(d, n, 2)
        c.check(RESID, SILU, c.run(RESID, T, num_sms=sms), T, f"{d}x{n} T={T} {want}-way global")


@pytest.mark.gpu
def test_unsupported_shapes_launch_nothing():
    """Return codes of calls the launcher rejects, with the output untouched: T = 0 and 257, n % 64 != 0, odd d, the TMA
    variant with n % 256 != 0, actStride not a multiple of 8, an unknown epilogue (3)."""
    ops = _ops()
    cl = ops.cuda_lib
    W = Experts(1, 256, 512, 3)
    w = W.device()
    act = torch.randn(257, 520, device="cuda").bfloat16()
    for what, epi, d, n, T, stride, variant, rc in [("T=0", F32, 256, 512, 0, 512, 0, -1), ("T=257", F32, 256, 512, 257, 512, 0, -1),
                                                    ("n=480", F32, 256, 480, 16, 512, 0, -1), ("d=255", F32, 255, 512, 16, 512, 0, -1),
                                                    ("tma n=320", F32, 256, 320, 16, 512, 2, -6),
                                                    ("actStride=516", F32, 256, 512, 16, 516, 0, -4), ("epi=3", 3, 256, 512, 16, 512, 0, -5)]:
        out = torch.full((260, 256), NAN_F32, dtype=torch.int32, device="cuda")
        p = ops.gemm_q40_tc_plan(epi, d, n, T, act_stride=stride, num_sms=_device_sms(), variant=["auto", "ldg", "tma"][variant])
        got = cl.lib().dl_gemm_q40_tc(epi, w.qs.data_ptr(), w.scales.data_ptr(), d, n, act.data_ptr(), stride, T, out.data_ptr(), 256,
                                      _device_sms(), SILU, cl.stream_ptr(), 0, variant)
        torch.cuda.synchronize()
        assert p.rc == rc and got == rc, f"{what}: plan rc {p.rc}, launch rc {got}, expected {rc}"
        assert (out == NAN_F32).all(), f"{what}: output written"


# ---- earlier cases, now against float64 ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ldg", "tma"])
@pytest.mark.parametrize("d,n,T", [(256, 256, 16), (128, 64, 1), (384, 512, 17), (6144, 4096, 64), (4096, 14336, 64),
                                   (1024, 1792, 200), (2048, 4096, 256), (1000, 2176, 33), (28672, 4096, 100), (4096, 4096, 192),
                                   (4096, 14336, 128)])
def test_gemm_store_f32(d, n, T, variant):
    if variant == "tma" and n % 256:
        pytest.skip("TMA-staged variant needs n % 256 == 0")
    c = case(d, n, 5)
    p = _ops().gemm_q40_tc_plan(F32, d, n, T, num_sms=_device_sms(), variant=variant)
    assert p.rc == 0 and p.kernel == (1 if variant == "ldg" else 2), p
    _note(_path(p), c.check(F32, SILU, c.run(F32, T, num_sms=_device_sms(), variant=variant), T, f"{d}x{n} T={T} {variant} {p}"))


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", ["1", "0"])
def test_gemm_split_k_over_token_tiles(cluster, monkeypatch):
    """2-way split-K over 2 token tiles (Llama-3.1-8B W2 rows halved, 128 tokens, 64 SMs), reduced inside a thread-block cluster or
    (cluster = 0) through the global scratch; residual epilogue."""
    monkeypatch.delenv("DL_GEMM_SPLITK", raising=False)
    monkeypatch.setenv("DL_GEMM_CLUSTER", cluster)
    d, n, T = 2048, 14336, 128
    _assert_plan(RESID, d, n, T, 64, "tma", (2, 2, int(cluster)))
    c = case(d, n, 8)
    _note((2, 2, int(cluster)), c.check(RESID, SILU, c.run(RESID, T, num_sms=64, variant="tma"), T, f"split-K cluster={cluster}"))


@pytest.mark.gpu
def test_gemm_residual_and_swiglu():
    c = case(1024, 1024, 6)
    for epi, act_fn in ((RESID, SILU), (SWIGLU, SILU), (SWIGLU, GELU)):
        c.check(epi, act_fn, c.run(epi, 48, num_sms=_device_sms(), act_fn=act_fn), 48, f"1024x1024 epi {epi} act {act_fn}")


@pytest.mark.gpu
def test_rmsnorm_bf16():
    """rmsNormBf16Kernel at the model dims with xStride = n + 12, bracketed against float64; w = None converts only (bitwise
    x.bfloat16())."""
    ops = _ops()
    g = gen("rmsnorm")
    for n in (1024, 4096, 5120, 8192):
        T = 37
        xb = torch.randn(T, n + 12, device="cuda", generator=g) * 3
        x = xb[:, :n]
        w = 1 + 0.1 * torch.randn(n, device="cuda", generator=g)
        y = ops.rmsnorm_bf16(x, w, 1e-5)
        xd = x.double()
        r = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-5)
        lo, hi = bf16_bracket(r, REL_NORM * r.abs())
        assert_bracketed(y, lo, hi, f"rmsnorm n={n}")
        assert torch.equal(ops.rmsnorm_bf16(x, None, 1e-5), x.bfloat16()), f"rmsnorm n={n}: w = None is not a plain conversion"
