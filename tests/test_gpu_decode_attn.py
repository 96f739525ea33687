"""Decode attention (csrc/cuda/attn_decode.cu) against a float64 reference, beyond the first KV split.

Kernels under test, through their stand-alone entry points:
* attnFusedKernel: QK-norm + RoPE + KV append + split-KV attention of one token; ceil(nPos / 64) splits, capped at nSplits.
* ropeKvKernel + attnDecodeKernel: the GEMV-path batch of up to 8 tokens; nSplits splits, those past nPos empty.
The persistent decode kernel's attention (mega_decode.cu) cannot be launched alone; the engine tests at the end of this file
cover it at long context.

The inputs are built so that a split that is lost or misweighted moves the output by far more than the tolerance: scores
with a standard deviation of about 4, random V rows, and "needle" keys parallel to q at split boundaries, at the last cached
row and at the new token.

Tolerance: both sides read the same bf16 cache, so the difference is the kernel's f32 arithmetic (fast __expf, online
softmax rescaling, split merge). The bound is 2e-4 * max|V| (plus one bf16 ulp of the reference for bf16 outputs). On an
H100 80GB HBM3 (700 W) the largest error over all cases is 0.48 of the bound, and that is the half-ulp rounding of the bf16
outputs. A merge that drops the last split errs by up to 5200x the bound, and a wrong GQA head mapping by up to 8800x;
a wrong rotary row moves the rotated q by about 10 (the bound there is 2e-5 of max|q|).
"""
import dataclasses
import hashlib
import math
import zlib

import numpy as np
import pytest
import torch

SEQ = 4096
TOL_V = 2e-4        # f32 output tolerance, in units of max|V| over the attended rows
NEEDLE_SCORE = 30.0  # scaled score of a cached needle key; random keys stay below ~16
EPS = 1e-6


# ---- float64 reference (runs on CPU or CUDA tensors) -------------------------------------------------------------------
def rope_table(hd: int, seq: int = SEQ) -> torch.Tensor:
    """[seq, hd/2, 2] f32 (cos, sin) table from the host builder, for a plain RoPE model with head dim `hd`."""
    from distributed_llama_b200 import host
    from distributed_llama_b200.formats import quants
    from distributed_llama_b200.formats.model_file import HEADER_KEYS
    from distributed_llama_b200.models.config import get_config
    cfg = dataclasses.replace(get_config("tiny-qwen3"), head_dim=hd, max_seq_len=seq, rope_theta=10000)
    H = host()
    hdr = H.parse_model_header(H.build_model_header([(HEADER_KEYS[k], v) for k, v in cfg.header_params(quants.F_Q40).items()]), 0, 0)
    return torch.from_numpy(np.asarray(H.build_rope_table(hdr, seq)).copy())


def ref_norm_rope(x: torch.Tensor, w, eps: float, cs: torch.Tensor) -> torch.Tensor:
    """Optional per-head RMS norm with weight `w`, then adjacent-pair rotation by the (cos, sin) row `cs` [hd/2, 2]."""
    x = x.double()
    if w is not None:
        x = w.double() * (x * torch.rsqrt(x.pow(2).mean(dim=-1, keepdim=True) + eps))
    c, s = cs[..., 0].double(), cs[..., 1].double()
    a, b = x[..., 0::2], x[..., 1::2]
    out = torch.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = a * s + b * c
    return out


def ref_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, p: int) -> torch.Tensor:
    """softmax(q . K[0..p]^T / sqrt(hd)) . V[0..p] per q-head; q-head h reads KV head h // (nHeads // nKvHeads).
    q [nHeads, hd] (already normalised and rotated); caches [nKvHeads, seq, hd] as stored. Returns f64 [nHeads, hd]."""
    n_heads, hd = q.shape
    n_kv = k_cache.shape[0]
    g = n_heads // n_kv
    K = k_cache[:, :p + 1].double()
    V = v_cache[:, :p + 1].double()
    s = torch.einsum("kgd,kpd->kgp", q.double().view(n_kv, g, hd), K) / math.sqrt(hd)
    return torch.einsum("kgp,kpd->kgd", torch.softmax(s, dim=-1), V).reshape(n_heads, hd)


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (8 significant bits)."""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def assert_row_close(got_bf16: torch.Tensor, want: torch.Tensor, what: str):
    """A bf16 cache row within one bf16 ulp of the float64 value. The kernel computes in f32 before rounding: where RoPE
    cancels to a value near zero, its f32 rounding error (below 2^-20 of the row's largest value) may exceed that ulp."""
    want = want.double()
    err = (got_bf16.double() - want).abs()
    bad = err > bf16_ulp(want) + 2.0 ** -20 * want.abs().max()
    assert not bad.any(), f"{what}: {int(bad.sum())} values off by more than 1 bf16 ulp (max err {err.max().item():.3g})"


def assert_out_close(got: torch.Tensor, ref: torch.Tensor, vmax: float, what: str, bf16: bool = False):
    tol = TOL_V * vmax + (bf16_ulp(ref) if bf16 else 0.0)
    err = (got.double() - ref).abs()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    ratio = (err / tol).max().item()
    assert ratio <= 1.0, f"{what}: max err {err.max().item():.3g} = {ratio:.3g} x tolerance (max|V| {vmax:.3g})"


def test_reference_helpers_on_cpu():
    """The reference helpers on CPU tensors: a needle parallel to q takes the softmax, RoPE preserves the norm."""
    torch.manual_seed(0)
    hd, n_kv, g = 64, 2, 3
    cs = rope_table(hd, 16)
    x = torch.randn(n_kv * g, hd)
    r = ref_norm_rope(x, None, EPS, cs[5])
    assert torch.allclose(r.norm(dim=-1), x.double().norm(dim=-1))
    k = torch.randn(n_kv, 16, hd).bfloat16()
    v = torch.randn(n_kv, 16, hd).bfloat16()
    k[1, 9] = (r[3] / r[3].norm() * NEEDLE_SCORE * math.sqrt(hd) / r[3].norm()).bfloat16()
    out = ref_attention(r, k, v, 12)
    assert torch.allclose(out[3], v[1, 9].double(), atol=1e-3)


# ---- harness ---------------------------------------------------------------------------------------------------------
TAIL = 64   # NaN-filled floats past the end of every scratch / output buffer


def _nan(n, dtype=torch.float32):
    return torch.full((n,), float("nan"), dtype=dtype, device="cuda")


class Scratch:
    """partial / counters buffers shared by consecutive launches, as the engine shares them."""

    def __init__(self, n_tok, n_heads, n_splits, hd):
        self.n_part = n_tok * n_heads * n_splits * (hd + 2)
        self.partial = _nan(self.n_part + TAIL)
        self.n_cnt = n_tok * n_heads
        self.counters = torch.zeros(self.n_cnt + TAIL, dtype=torch.int32, device="cuda")
        self.counters[self.n_cnt:] = 0x7eadbeef

    def check(self, what):
        assert torch.isnan(self.partial[self.n_part:]).all(), f"{what}: partial written past its end"
        assert (self.counters[:self.n_cnt] == 0).all(), f"{what}: split counters not reset"
        assert (self.counters[self.n_cnt:] == 0x7eadbeef).all(), f"{what}: counters written past their end"


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _eff_fused(p, n_splits):
    return max(1, min((p + 64) // 64, n_splits))


def _needles(p, eff):
    """Needle rows: none (-1), position 0, the first and last row of an interior split, the last cached row, the new row."""
    nPos = p + 1
    chunk = -(-nPos // eff)
    rows = [-1, 0, p - 1, p]
    if eff >= 2:
        b = (eff // 2) * chunk
        rows += [b, b - 1]
    seen, out = set(), []
    for r in rows:
        if r not in seen and -1 <= r <= p:
            seen.add(r)
            out.append(r)
    return out


def _case_inputs(n_heads, n_kv, hd, qk_norm, n_tok, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    qkv = torch.randn(n_tok, q_dim + 2 * kv_dim, device="cuda", generator=g)
    if qk_norm:
        # normalised q has rms |w_q| ~ 4: score std ~ 4 against unit-variance cached keys
        qkv *= 3.0
        qn = 4.0 * (1.0 + 0.1 * torch.randn(hd, device="cuda", generator=g))
        kn = 1.0 + 0.1 * torch.randn(hd, device="cuda", generator=g)
    else:
        qkv[:, :q_dim] *= 4.0
        qn = kn = None
    k_cache = torch.randn(n_kv, SEQ, hd, device="cuda", generator=g).bfloat16()
    v_cache = torch.randn(n_kv, SEQ, hd, device="cuda", generator=g).bfloat16()
    return qkv, qn, kn, k_cache, v_cache


def _plant_cached_needle(k_cache, q_rot, row, g):
    """K[kvh, row] parallel to the (rotated) q of the first q-head of every KV group, at scaled score NEEDLE_SCORE."""
    n_kv, _, hd = k_cache.shape
    for kvh in range(n_kv):
        qh = q_rot[kvh * g]
        k_cache[kvh, row] = (qh / qh.norm() * (NEEDLE_SCORE * math.sqrt(hd) / qh.norm())).bfloat16()


def _plant_new_needle(qkv_row, n_heads, n_kv, hd):
    """The new token's raw k equals the raw q of the first q-head of its group."""
    g = n_heads // n_kv
    q_dim = n_heads * hd
    for kvh in range(n_kv):
        qkv_row[q_dim + kvh * hd: q_dim + (kvh + 1) * hd] = qkv_row[kvh * g * hd: (kvh * g + 1) * hd]


# ---- attnFusedKernel -------------------------------------------------------------------------------------------------
_ROPE = {}


def _rope(hd):
    if hd not in _ROPE:
        _ROPE[hd] = rope_table(hd).cuda()
    return _ROPE[hd]


def _run_fused(lib, cl, qkv_row, p, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, out):
    pos = torch.tensor([p], dtype=torch.int32, device="cuda")
    rc = lib.dl_attn_fused(qkv_row.data_ptr(), pos.data_ptr(), _rope(hd).data_ptr(), qn.data_ptr() if qn is not None else None,
                           kn.data_ptr() if kn is not None else None, EPS, k_cache.data_ptr(), v_cache.data_ptr(),
                           n_heads, n_kv, hd, SEQ, n_splits, scr.partial.data_ptr(), scr.counters.data_ptr(), out.data_ptr(),
                           cl.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()


def _fused_once(lib, cl, qkv_row, p, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, what):
    """One launch at position p, checked against the reference and for side effects. Leaves the kernel's row p in the cache."""
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    cs = _rope(hd)[p]
    k_before, v_before, qkv_before = k_cache.clone(), v_cache.clone(), qkv_row.clone()
    out = _nan(q_dim + TAIL)
    _run_fused(lib, cl, qkv_row, p, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, out)
    # side effects: only row p of every KV head changes, to the bf16 of the rotated k and of v
    assert torch.equal(qkv_row, qkv_before), f"{what}: qkv modified"
    k_new = ref_norm_rope(qkv_row[q_dim:q_dim + kv_dim].view(n_kv, hd), kn, EPS, cs)
    v_new = qkv_row[q_dim + kv_dim:].view(n_kv, hd).double()
    assert_row_close(k_cache[:, p], k_new, f"{what}: k row {p}")
    assert_row_close(v_cache[:, p], v_new, f"{what}: v row {p}")
    for c, before in ((k_cache, k_before), (v_cache, v_before)):
        mask = torch.ones(SEQ, dtype=torch.bool, device="cuda")
        mask[p] = False
        assert torch.equal(c[:, mask], before[:, mask]), f"{what}: cache rows other than {p} changed"
    scr.check(what)
    assert torch.isnan(out[q_dim:]).all(), f"{what}: output written past its end"
    # attention over the cache as it now stands: rows < p as given, row p as the kernel rounded it (checked above)
    q_rot = ref_norm_rope(qkv_row[:q_dim].view(n_heads, hd), qn, EPS, cs)
    ref = ref_attention(q_rot, k_cache, v_cache, p)
    vmax = v_cache[:, :p + 1].float().abs().max().item()
    assert_out_close(out[:q_dim].view(n_heads, hd), ref, vmax, what)


def _fused_case(n_heads, n_kv, hd, qk_norm, p, n_splits):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    seed = _seed(n_heads, n_kv, hd, qk_norm, p, n_splits)
    qkv, qn, kn, k_cache, v_cache = _case_inputs(n_heads, n_kv, hd, qk_norm, 1, seed)
    q_dim = n_heads * hd
    g = n_heads // n_kv
    scr = Scratch(1, n_heads, n_splits, hd)
    q_rot = ref_norm_rope(qkv[0, :q_dim].view(n_heads, hd), qn, EPS, _rope(hd)[p])
    k0 = k_cache.clone()
    for row in _needles(p, _eff_fused(p, n_splits)):
        k_cache.copy_(k0)
        row_qkv = qkv[0].clone()
        if row == p:
            _plant_new_needle(row_qkv, n_heads, n_kv, hd)
        elif row >= 0:
            _plant_cached_needle(k_cache, q_rot, row, g)
        what = f"fused ({n_heads},{n_kv},{hd}) norm={qk_norm} p={p} nSplits={n_splits} needle={row}"
        _fused_once(lib, cl, row_qkv, p, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, what)


FUSED_POSITIONS = [0, 1, 63, 64, 65, 127, 128, 255, 256, 257, 1000, 2047, 4095]


@pytest.mark.gpu
@pytest.mark.parametrize("n_splits", [1, 3, 8, 32])
@pytest.mark.parametrize("p", FUSED_POSITIONS)
@pytest.mark.parametrize("qk_norm", [False, True])
@pytest.mark.parametrize("n_heads,n_kv,hd", [(32, 8, 128), (6, 2, 64)])
def test_attn_fused_position_sweep(n_heads, n_kv, hd, qk_norm, p, n_splits):
    _fused_case(n_heads, n_kv, hd, qk_norm, p, n_splits)


@pytest.mark.gpu
@pytest.mark.parametrize("n_splits", [3, 32])
@pytest.mark.parametrize("p", [1, 65, 257, 2047, 4095])
@pytest.mark.parametrize("qk_norm", [False, True])
@pytest.mark.parametrize("n_heads,n_kv,hd", [(40, 8, 128), (8, 8, 128), (4, 1, 128), (32, 8, 64)])
def test_attn_fused_head_shapes(n_heads, n_kv, hd, qk_norm, p, n_splits):
    _fused_case(n_heads, n_kv, hd, qk_norm, p, n_splits)


@pytest.mark.gpu
@pytest.mark.parametrize("n_splits", [3, 32])
@pytest.mark.parametrize("n_heads,n_kv,hd,qk_norm", [(32, 8, 128, False), (6, 2, 64, True)])
def test_attn_fused_back_to_back(n_heads, n_kv, hd, qk_norm, n_splits):
    """Launches on shared partial/counter buffers at positions that change the effective split count: a stale counter or
    partial from the previous launch would show up in the next one's output."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    qkv, qn, kn, k_cache, v_cache = _case_inputs(n_heads, n_kv, hd, qk_norm, 1, 99 + n_splits)
    scr = Scratch(1, n_heads, n_splits, hd)
    for i, p in enumerate([63, 64, 65, 257, 64, 4095, 1, 2047, 128]):
        row_qkv = qkv[0] * (1.0 + 0.01 * i)
        _fused_once(lib, cl, row_qkv, p, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr,
                    f"fused back-to-back #{i} p={p} nSplits={n_splits}")


# ---- ropeKvKernel + attnDecodeKernel ----------------------------------------------------------------------------------
def _run_rope(lib, cl, qkv, pos, qn, kn, k_cache, v_cache, n_heads, n_kv, hd):
    rc = lib.dl_rope_kv(qkv.data_ptr(), qkv.shape[1], pos.data_ptr(), _rope(hd).data_ptr(), qn.data_ptr() if qn is not None else None,
                        kn.data_ptr() if kn is not None else None, EPS, n_heads, n_kv, hd, SEQ, k_cache.data_ptr(), v_cache.data_ptr(),
                        qkv.shape[0], cl.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()


def _rope_checked(lib, cl, qkv, positions, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, what):
    """ropeKvKernel on nb tokens: q rotated in place, k/v rows of the given (distinct) positions written, nothing else touched.
    Returns the float64 rotated q [nb, nHeads, hd]."""
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    nb = len(positions)
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    k_before, v_before, qkv_before = k_cache.clone(), v_cache.clone(), qkv.clone()
    _run_rope(lib, cl, qkv, pos, qn, kn, k_cache, v_cache, n_heads, n_kv, hd)
    q_rot = torch.stack([ref_norm_rope(qkv_before[t, :q_dim].view(n_heads, hd), qn, EPS, _rope(hd)[p]) for t, p in enumerate(positions)])
    err = (qkv[:, :q_dim].view(nb, n_heads, hd).double() - q_rot).abs().max().item()
    assert err <= 2e-5 * q_rot.abs().max().item(), f"{what}: rotated q off by {err:.3g}"
    assert torch.equal(qkv[:, q_dim:], qkv_before[:, q_dim:]), f"{what}: k/v columns of qkv modified"
    mask = torch.ones(SEQ, dtype=torch.bool, device="cuda")
    for t, p in enumerate(positions):
        mask[p] = False
        k_new = ref_norm_rope(qkv_before[t, q_dim:q_dim + kv_dim].view(n_kv, hd), kn, EPS, _rope(hd)[p])
        assert_row_close(k_cache[:, p], k_new, f"{what}: k row {p}")
        assert_row_close(v_cache[:, p], qkv_before[t, q_dim + kv_dim:].view(n_kv, hd), f"{what}: v row {p}")
    for c, before in ((k_cache, k_before), (v_cache, v_before)):
        assert torch.equal(c[:, mask], before[:, mask]), f"{what}: cache rows other than {positions} changed"
    return q_rot


@pytest.mark.gpu
@pytest.mark.parametrize("qk_norm", [False, True])
@pytest.mark.parametrize("n_heads,n_kv,hd", [(32, 8, 128), (6, 2, 64), (8, 2, 256)])
def test_rope_kv(n_heads, n_kv, hd, qk_norm):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    qkv, qn, kn, k_cache, v_cache = _case_inputs(n_heads, n_kv, hd, qk_norm, 8, hd + qk_norm)
    for positions in ([0, 1, 2, 3, 4, 5, 6, 7], [4088, 4089, 4090, 4091, 4092, 4093, 4094, 4095], [1000, 3, 4095, 64, 257, 63, 2047, 9]):
        _rope_checked(lib, cl, qkv.clone(), positions, qn, kn, k_cache, v_cache, n_heads, n_kv, hd,
                      f"rope ({n_heads},{n_kv},{hd}) norm={qk_norm} pos={positions[0]}..")


def _decode_case(lib, cl, qkv, positions, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, bf16_out, what):
    """ropeKvKernel then attnDecodeKernel over nb tokens, as the engine runs a GEMV-path batch; checks the output against the
    reference and the side effects. Columns past qDim of the output rows must stay untouched."""
    q_dim = n_heads * hd
    nb = len(positions)
    q_rot = _rope_checked(lib, cl, qkv, positions, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, what)
    out_stride = q_dim + 40
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    dt = torch.bfloat16 if bf16_out else torch.float32
    out = _nan(nb * out_stride + TAIL, dt)
    k_before, v_before = k_cache.clone(), v_cache.clone()
    rc = lib.dl_attn_decode(qkv.data_ptr(), qkv.shape[1], pos.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), n_heads, n_kv, hd, SEQ,
                            n_splits, scr.partial.data_ptr(), scr.counters.data_ptr(), None if bf16_out else out.data_ptr(), out_stride,
                            out.data_ptr() if bf16_out else None, nb, cl.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(k_cache, k_before) and torch.equal(v_cache, v_before), f"{what}: attention wrote the cache"
    scr.check(what)
    rows = out[:nb * out_stride].view(nb, out_stride)
    assert torch.isnan(rows[:, q_dim:]).all() and torch.isnan(out[nb * out_stride:]).all(), f"{what}: output written past qDim"
    for t, p in enumerate(positions):
        ref = ref_attention(q_rot[t], k_cache, v_cache, p)
        vmax = v_cache[:, :p + 1].float().abs().max().item()
        assert_out_close(rows[t, :q_dim].view(n_heads, hd), ref, vmax, f"{what}: token {t} (p={p})", bf16=bf16_out)


DECODE_BATCHES = [(nb, p0) for nb in (1, 2, 4, 8) for p0 in (0, 61, SEQ - nb)] + [(4, None), (8, None)]
_UNRELATED = {4: [1000, 3, 4095, 64], 8: [1000, 3, 4095, 64, 257, 0, 2047, 129]}


@pytest.mark.gpu
@pytest.mark.parametrize("bf16_out", [False, True])
@pytest.mark.parametrize("n_splits", [1, 7, 32])
@pytest.mark.parametrize("nb,p0", DECODE_BATCHES)
@pytest.mark.parametrize("n_heads,n_kv,hd,qk_norm", [(32, 8, 128, False), (6, 2, 64, True)])
def test_attn_decode_batch(n_heads, n_kv, hd, qk_norm, nb, p0, n_splits, bf16_out):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    positions = list(range(p0, p0 + nb)) if p0 is not None else _UNRELATED[nb]
    seed = _seed(n_heads, hd, nb, p0, n_splits, bf16_out)
    qkv, qn, kn, k_cache, v_cache = _case_inputs(n_heads, n_kv, hd, qk_norm, nb, seed)
    q_dim = n_heads * hd
    g = n_heads // n_kv
    scr = Scratch(nb, n_heads, n_splits, hd)
    t_last = max(range(nb), key=lambda t: positions[t])
    P = positions[t_last]
    q_rot = ref_norm_rope(qkv[t_last, :q_dim].view(n_heads, hd), qn, EPS, _rope(hd)[P])
    k0 = k_cache.clone()
    for row in _needles(P, n_splits):
        k_cache.copy_(k0)
        batch = qkv.clone()
        if row in positions:
            if row != P:
                continue     # a row this batch writes: only the last token's own row is planted (as its raw k)
            _plant_new_needle(batch[t_last], n_heads, n_kv, hd)
        elif row >= 0:
            _plant_cached_needle(k_cache, q_rot, row, g)
        what = f"decode ({n_heads},{n_kv},{hd}) norm={qk_norm} pos={positions} nSplits={n_splits} bf16={bf16_out} needle={row}"
        _decode_case(lib, cl, batch, positions, qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, bf16_out, what)


@pytest.mark.gpu
@pytest.mark.parametrize("n_splits", [7, 32])
def test_attn_decode_back_to_back(n_splits):
    """Single-token launches on shared scratch at positions that change how many splits are non-empty."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    n_heads, n_kv, hd = 32, 8, 128
    qkv, qn, kn, k_cache, v_cache = _case_inputs(n_heads, n_kv, hd, False, 1, 7 + n_splits)
    scr = Scratch(1, n_heads, n_splits, hd)
    for i, p in enumerate([63, 64, 65, 257, 64, 3, 4095, 0, 31]):
        _decode_case(lib, cl, qkv * (1.0 + 0.01 * i), [p], qn, kn, k_cache, v_cache, n_heads, n_kv, hd, n_splits, scr, i % 2 == 1,
                     f"decode back-to-back #{i} p={p} nSplits={n_splits}")


# ---- synthetic model files with sharper attention -----------------------------------------------------------------------
# sha256 of the default files (seed 7): attn_gain must not change what the other tests run on
_DEFAULT_FILES = {"tiny-llama31": "cceaf39573320790ecfcee9cefd2aa7bbcd5a09d9d0c259bd876028d7b0a64c8",
                  "tiny-qwen3": "50717eb831bc79b00dfa86915db090a382ad5b70e3c19264d2eeaac9ea6aca68"}


def test_synthetic_attn_gain(tmp_path):
    from distributed_llama_b200.formats import ModelFile, quants
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    for name, digest in _DEFAULT_FILES.items():
        p = tmp_path / f"{name}.m"
        write_synthetic_model(str(p), get_config(name), seed=7)
        assert hashlib.sha256(p.read_bytes()).hexdigest() == digest, name
        write_synthetic_model(str(p), get_config(name), seed=7, attn_gain=1.0)
        assert hashlib.sha256(p.read_bytes()).hexdigest() == digest, name
        # f32 weights: the gain scales exactly the tensors that set the score scale, and nothing else
        a, b = tmp_path / f"{name}-1.m", tmp_path / f"{name}-2.m"
        write_synthetic_model(str(a), get_config(name), weights_float_type=quants.F_32, seed=7)
        write_synthetic_model(str(b), get_config(name), weights_float_type=quants.F_32, seed=7, attn_gain=2.0)
        ma, mb = ModelFile(str(a)), ModelFile(str(b))
        scaled = ("block_norm_q", "block_norm_k") if ma.header.qk_norm else ("block_matmul_q", "block_matmul_k")
        for t in ("block_matmul_q", "block_matmul_k", "block_matmul_v", "block_matmul_wo", "block_norm_0") + \
                 (("block_norm_q", "block_norm_k") if ma.header.qk_norm else ()):
            x, y = (m.tensor_f32(m.entry(t, 1)) for m in (ma, mb))
            np.testing.assert_array_equal(y, 2 * x if t in scaled else x, err_msg=f"{name} {t}")


# ---- engine: persistent kernel, fused kernel and GEMV-path attention at long context -----------------------------------
PROMPT_LEN = 1925    # 10 tensor-core chunks of 192, then a GEMV batch of 4 and one single-token step


@pytest.fixture(scope="module")
def long_models(tmp_path_factory):
    """tiny-llama31 (head dim 64) and tiny-qwen3 (head dim 128, QK-norm) with a 4096-token context and attention scores
    four times as large as the default files."""
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    root = tmp_path_factory.mktemp("long_models")
    out = {}
    for name in ("tiny-llama31", "tiny-qwen3"):
        path = str(root / f"{name}-4k.m")
        write_synthetic_model(path, dataclasses.replace(get_config(name), max_seq_len=SEQ), seed=7, attn_gain=2.0)
        out[name] = path
    return out


def _prompt():
    return [(7 * i + 3) % 500 + 1 for i in range(PROMPT_LEN)]


def _engine(path, **kw):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    return Engine(load_device_weights(ModelFile(path)), **kw)


def _copy_caches(dst, src):
    for d, s in zip(dst.k_cache + dst.v_cache, src[0] + src[1]):
        d.copy_(s)


@pytest.mark.gpu
@pytest.mark.parametrize("n_splits", [0, 3])
@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_engine_long_context_decode_paths(long_models, monkeypatch, name, n_splits):
    """Chunked prefill of 1925 tokens against the oracle; then one step at positions 1925, 2047 and 4095 through the
    persistent kernel, the fused kernel and the rope + split-KV kernels over identical caches. On a 132-SM H100 with the
    default split count they merge 8, 31 and 32 splits at 1926 positions; n_splits=3 caps all three."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.reference import OracleModel
    path = long_models[name]
    eng = _engine(path, n_splits=n_splits)
    oracle = OracleModel(ModelFile(path), act_quant="q80", device="cuda")
    toks = _prompt()
    ref = oracle.forward(toks, 0)[-1]
    lg = eng.prefill(toks, 0).clone()
    err = (lg - ref).abs().max().item()
    assert err < 0.12, f"prefill: {err}"
    saved = ([c.clone() for c in eng.k_cache], [c.clone() for c in eng.v_cache])
    o_saved = ([c.clone() for c in oracle.k_cache], [c.clone() for c in oracle.v_cache])
    monkeypatch.setenv("DL_NO_FUSED_ATTN", "1")
    eng_s = _engine(path, n_splits=n_splits)
    monkeypatch.delenv("DL_NO_FUSED_ATTN")
    eng_s.enable_mega(False)
    _copy_caches(eng_s, saved)
    for pos in (PROMPT_LEN, 2047, SEQ - 1):
        tok = 11
        _copy_caches(oracle, o_saved)
        want = oracle.forward([tok], pos)[0]
        got = {}
        _copy_caches(eng, saved)
        eng.enable_mega(True)
        got["persistent"] = eng.step(tok, pos).clone()
        assert eng.mega_active
        _copy_caches(eng, saved)
        eng.enable_mega(False)
        got["fused"] = eng.step(tok, pos).clone()
        _copy_caches(eng_s, saved)
        got["split-kv"] = eng_s.step(tok, pos).clone()
        for k, v in got.items():
            err = (v - want).abs().max().item()
            assert err < 0.12, f"{k} vs oracle at pos {pos}: {err}"
        for k in ("fused", "split-kv"):
            err = (got[k] - got["persistent"]).abs().max().item()
            assert err < 2e-3, f"{k} vs persistent at pos {pos}: {err}"


@pytest.mark.gpu
@pytest.mark.parametrize("mega", [True, False])
@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_engine_long_context_graph_replay(long_models, name, mega):
    """One captured decode graph replayed from position 250 and from 2040: the split count is chosen on the device, so the
    replays cross the 256- and 64-position split boundaries. Greedy tokens must equal those of eager launches."""
    eng = _engine(long_models[name])
    eng.enable_mega(mega)
    toks = _prompt()
    eng.prefill(toks, 0, want_logits=False)
    saved = ([c.clone() for c in eng.k_cache], [c.clone() for c in eng.v_cache])
    out = {}
    for use_graph in (True, False):
        for start in (250, 2040):
            _copy_caches(eng, saved)
            out[use_graph, start] = eng.decode_greedy(toks[start] if start < PROMPT_LEN else 11, start, 24, use_graph=use_graph)
            assert eng.mega_active == mega
    for start in (250, 2040):
        assert out[True, start] == out[False, start], start
