"""Float64 reference helpers shared by the q40 matrix tests (tests/test_gpu_gemm_tc.py, tests/test_gpu_moe.py, tests/test_gpu_gemv.py)
and the model-level tests (tests/test_gpu_mega_shapes.py, tests/test_gpu_prefill_chain.py, tests/test_gpu_moe_chain.py).

* Random q40 matrices as raw 18-byte blocks (f16 scale + 16 bytes of nibbles) and their device layout.
* The weights the tensor-core dequant warps build from them: rn_bf16(rn_bf16(f16 scale) * (q - 8)).
* The q80 grid of decode activations, with the ambiguity of a rounding whose input is only known within an interval.
* Checks of a kernel's values against a float64 reference with a per-element bound, or against the bf16 roundings of the two ends
  of an interval.
* Engine-level pieces of the model tests (test_gpu_prefill_chain.py, test_gpu_batched_steps.py): random K/V caches with NaN rows,
  the caches as the attention kernels read them, the stored K/V rows against float64, and the per-stage error / bound report.
"""
import math
import zlib

import numpy as np
import torch

U = 2.0 ** -24                   # unit roundoff of f32
REL_NORM = 2.0 ** -18
CONTROL_MIN = 10.0


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def gen(*key):
    return torch.Generator(device="cuda").manual_seed(seed_of(*key))


# ---- q40 blocks ------------------------------------------------------------------------------------------------------------
def q40_parts(raw, rows, n):
    """raw: uint8 [rows * n / 32][18] blocks of a [rows][n] matrix -> (f16 scales [rows][n / 32], q - 8 as float64 [rows][n]).
    Within a block the low nibbles of the 16 bytes are elements 0..15 and the high nibbles elements 16..31."""
    blk = n // 32
    sc = raw[:, :2].contiguous().view(torch.float16).view(rows, blk)
    lo = (raw[:, 2:] & 15).double() - 8
    hi = (raw[:, 2:] >> 4).double() - 8
    q = torch.cat([lo, hi], dim=1).view(rows, n)
    return sc, q


def w_tc_of(sc, q):
    """Weights as the tensor-core dequant builds them: rn_bf16(rn_bf16(f16 scale) * (q - 8)), as float64."""
    sb = sc.float().bfloat16().float().repeat_interleave(32, dim=1)
    return (sb * q.float()).bfloat16().double()


def q40_exact(raw, rows, n):
    """raw blocks of a [rows][n] matrix dequantised exactly (the decode GEMV's weights), f64 [rows][n], and |w| + 8 |scale| (its
    f32 error scale: the GEMV multiplies unsigned nibbles and subtracts 8 x scale x sum(q) afterwards)."""
    sc, q = q40_parts(raw, rows, n)
    s = sc.double().repeat_interleave(32, dim=1)
    return s * q, s.abs() * (q.abs() + 8)


def q40_tc(raw, rows, n):
    """raw blocks of a [rows][n] matrix as the tensor-core dequant builds it (w_tc_of), f64."""
    return w_tc_of(*q40_parts(raw, rows, n))


class Experts:
    """E stacked random q40 matrices [rows][n] (raw 18-byte blocks + the device layout). Row r of matrix e is stack row e * rows + r.
    Scales are +-(0.5 .. 1.5) / (4 sqrt(n)), so a dot product with unit-variance activations is of order 1."""

    def __init__(self, E, rows, n, seed):
        g = gen("q40", E, rows, n, seed)
        nb = E * rows * n // 32
        sc = (torch.rand(nb, device="cuda", generator=g) + 0.5) / (4.0 * math.sqrt(n))
        sc = torch.where(torch.rand(nb, device="cuda", generator=g) < 0.5, -sc, sc).half()
        self.raw = torch.empty(nb, 18, dtype=torch.uint8, device="cuda")
        self.raw[:, :2] = sc.view(torch.uint8).view(nb, 2)
        self.raw[:, 2:] = torch.randint(0, 256, (nb, 16), dtype=torch.uint8, device="cuda", generator=g)
        self.E, self.rows, self.n = E, rows, n
        self._dev = {}

    def device(self, first=0, count=None):
        """DeviceQ40 of matrices [first, first + count) only (an expert-parallel rank's weights)."""
        from distributed_llama_b200.ops import DeviceQ40, repack_q40
        count = self.E - first if count is None else count
        if (first, count) not in self._dev:
            r0, nr = first * self.rows, count * self.rows
            dst = DeviceQ40.empty(nr, self.n)
            blk = self.n // 32
            repack_q40(self.raw[r0 * blk:(r0 + nr) * blk].reshape(-1), nr, self.n, dst)
            self._dev[first, count] = dst
        return self._dev[first, count]

    def _raw(self, e):
        blk = self.n // 32
        return self.raw[e * self.rows * blk:(e + 1) * self.rows * blk]

    def w_exact(self, e):
        """Matrix e dequantised exactly (q40_exact)."""
        return q40_exact(self._raw(e), self.rows, self.n)

    def w_tc(self, e=0):
        """Matrix e as the tensor-core dequant builds it."""
        return q40_tc(self._raw(e), self.rows, self.n)


# ---- comparisons ---------------------------------------------------------------------------------------------------------
def f64_to_bf16(x):
    """bf16 rounding of f64 values (via f32, as the kernels round their f32 values)."""
    return x.float().bfloat16().double()


def bf16_bracket(r, e):
    """bf16 roundings of the interval ends [r - e, r + e]: a value the kernel rounds from inside the interval lies between them."""
    return f64_to_bf16(r - e), f64_to_bf16(r + e)


def assert_within(got, ref, tol, what):
    """|got - ref| <= tol element-wise; returns the largest err / tol."""
    got = got.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err = (got - ref).abs()
    ratio = (err / tol.clamp_min(1e-30)).max().item()
    assert ratio <= 1.0, f"{what}: max err {err.max().item():.3g} = {ratio:.3g} x bound (max|ref| {ref.abs().max().item():.3g})"
    return ratio


def assert_bracketed(got, lo, hi, what):
    got = got.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    bad = (got < lo) | (got > hi)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} values outside the rounding interval "
                           f"(max distance {torch.maximum(lo - got, got - hi).max().item():.3g})")


# ---- decode activations --------------------------------------------------------------------------------------------------
C_SILU = 2.0 ** -19    # SiLU with __expf and fast division, relative


def q80_ref(v, rel):
    """q80 grid of f64 activations v [..., n] (blocks of 32: d = f16(amax / 127), q = rint(x / d)) and, per element, the most the
    kernel's grid value can differ when its input is within `rel` (relative) of v."""
    shp = v.shape
    g = v.reshape(-1, 32)
    d = g.abs().amax(1, keepdim=True) / 127.0

    def f16(t):
        return t.float().half().double()

    dq, dlo, dhi = f16(d), f16(d * (1 - rel)), f16(d * (1 + rel))
    t = torch.where(d > 0, g / d.clamp_min(1e-300), torch.zeros_like(g))
    q, qlo, qhi = torch.round(t), torch.round(t - t.abs() * rel), torch.round(t + t.abs() * rel)
    a = q * dq
    amb = torch.stack([(x * y - a).abs() for x in (qlo, qhi) for y in (dlo, dhi)]).amax(0)
    return a.reshape(shp), amb.reshape(shp)


def silu(x):
    return x / (1.0 + torch.exp(-x))


def swiglu_ref(gu, e_gu):
    """h = silu(gate) * up from interleaved rows (gate even, up odd) and the bound on the kernel's f32 h."""
    g, u, eg, eu = gu[..., 0::2], gu[..., 1::2], e_gu[..., 0::2], e_gu[..., 1::2]
    s = silu(g)
    h = s * u
    # |d silu / dx| <= 1.1
    return h, 1.1 * eg * u.abs() + s.abs() * eu + 1.1 * eg * eu + C_SILU * h.abs()


# ---- model-level float64 reference (a synthetic model file's q40 matrices; q80 decode activations with their ties) -----------
def _interleave_perm(hd):
    perm = np.empty(hd, dtype=np.int64)
    perm[0::2] = np.arange(hd // 2)
    perm[1::2] = np.arange(hd // 2) + hd // 2
    return torch.from_numpy(perm)


def dequant(raw):
    """q40 file rows [d, n/32, 18] -> (f32 values [d, n] (exact), f32 block scales [d, n/32])."""
    d = raw[..., :2].contiguous().view(torch.float16).float()        # [d, nb, 1]
    qs = raw[..., 2:].to(torch.int16)
    w = torch.cat([(qs & 15) - 8, (qs >> 4) - 8], -1).float().mul_(d)
    return w.view(raw.shape[0], -1), d.view(raw.shape[0], -1)


class Ref:
    """The model file's q40 matrices as raw file rows on the device, in the engine's row order (q|k|v rows concatenated, q and k rows
    in adjacent-pair RoPE order for NeoX models, w1/w3 rows interleaved); `gemv` dequantises them chunk by chunk. Mixture-of-experts
    files: the f32 router gate ("moe_gate", [E][dim]) and every expert's w13 / w2 stacked on a leading expert index, dequantised per
    expert on demand by expert_exact and expert_tc."""

    def __init__(self, path):
        from distributed_llama_b200 import host
        from distributed_llama_b200.formats import ModelFile
        from distributed_llama_b200.models.config import ROPE_FALCON
        self.mf = mf = ModelFile(path)
        self.h = h = mf.header
        self.hd, self.nh, self.nkv, self.dim, self.ff = h.head_dim, h.n_heads, h.n_kv_heads, h.dim, h.ff_dim
        self.q_dim, self.kv_dim = self.nh * self.hd, self.nkv * self.hd
        self.eps = float(h.norm_epsilon)
        perm = _interleave_perm(self.hd).cuda() if h.rope_type == ROPE_FALCON else None

        def heads(t, n_heads):
            return t if perm is None else t.view(n_heads, self.hd, *t.shape[1:])[:, perm].reshape(t.shape)

        def vec(name, l=0):
            return torch.from_numpy(np.array(mf.tensor_f32(mf.entry(name, l)))).cuda().double()

        self.n_experts, self.k = h.n_experts, h.n_active_experts
        self.layers = []
        for l in range(h.n_layers):
            q, k, v = (self._q40(n, l) for n in ("block_matmul_q", "block_matmul_k", "block_matmul_v"))
            L = dict(qkv=torch.cat([heads(q, self.nh), heads(k, self.nkv), v]), wo=self._q40("block_matmul_wo", l),
                     norm0=vec("block_norm_0", l), norm1=vec("block_norm_1", l), q_norm=None, k_norm=None)
            if self.n_experts:
                # per expert, as the engine holds them: w13 [E][2 ff][dim / 32][18] (gate / up rows interleaved), w2 [E][dim][ff / 32][18]
                L["moe_gate"] = torch.from_numpy(np.array(mf.tensor_f32(mf.entry("block_moe_gate", l)))).cuda().double().view(
                    self.n_experts, self.dim)
                L["w13"] = torch.stack([torch.stack([self._q40("block_matmul_w1", l, e), self._q40("block_matmul_w3", l, e)], 1)
                                        .reshape(2 * self.ff, self.dim // 32, 18) for e in range(self.n_experts)])
                L["w2"] = torch.stack([self._q40("block_matmul_w2", l, e) for e in range(self.n_experts)])
            else:
                w1, w3 = self._q40("block_matmul_w1", l), self._q40("block_matmul_w3", l)
                L["w13"] = torch.stack([w1, w3], 1).reshape(2 * self.ff, self.dim // 32, 18)
                L["w2"] = self._q40("block_matmul_w2", l)
                del w1, w3
            del q, k, v
            if h.qk_norm:
                L["q_norm"], L["k_norm"] = vec("block_norm_q", l), vec("block_norm_k", l)
                if perm is not None:
                    L["q_norm"], L["k_norm"] = L["q_norm"][perm], L["k_norm"][perm]
            self.layers.append(L)
        self.final_norm = vec("final_norm")
        self.wcls = self._q40("final_matmul_logits")
        self.rope = torch.from_numpy(np.asarray(host().build_rope_table(h, h.seq_len))).cuda().double()   # [seq, hd/2, (cos, sin)]

    def _q40(self, name, l=0, expert=0):
        e = self.mf.entry(name, l, expert)
        return torch.from_numpy(np.array(self.mf.raw(e))).cuda().view(e.d, e.n // 32, 18)

    def expert_exact(self, l, name, e):
        """MoE file: expert e's "w13" or "w2" of layer l dequantised exactly (q40_exact)."""
        raw = self.layers[l][name][e]
        return q40_exact(raw.reshape(-1, 18), raw.shape[0], raw.shape[1] * 32)

    def expert_tc(self, l, name, e):
        """MoE file: expert e's "w13" or "w2" of layer l as the tensor-core dequant builds it (q40_tc), bf16 [rows][n] (exact)."""
        raw = self.layers[l][name][e]
        return q40_tc(raw.reshape(-1, 18), raw.shape[0], raw.shape[1] * 32).bfloat16()

    def embedding(self, tok):
        e = self.mf.entry("embedding")
        row = np.array(self.mf.data[e.offset + tok * self.dim * 4: e.offset + (tok + 1) * self.dim * 4]).view(np.float32)
        return torch.from_numpy(row).cuda().double()


def rms(x, w, eps):
    return w * (x / torch.sqrt((x * x).mean(-1, keepdim=True) + eps))


def rope(x, row):
    """Adjacent-pair rotation of the rows of x [.., hd] by a rotary table row [hd/2, (cos, sin)]."""
    a, b = x[..., 0::2], x[..., 1::2]
    c, s = row[:, 0], row[:, 1]
    out = torch.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = a * s + b * c
    return out


def q80(v, tol=None, normed=False):
    """q80 round trip of the float64 vector v, as the kernel's prologue rounds it (d = fp16(amax / 127), q = rn(v / d)), with the
    alternatives the kernel may take instead. tol: absolute uncertainty of the kernel's input to this prologue (per element, 0 when
    the input is the kernel's own observed vector). normed: an RMS-norm prologue, whose f32 norm factor scales the whole vector.
    Returns (xq, alt): one row of alt per alternative the kernel may take instead, holding the change of xq it makes: one grid
    step of element i where i lies within the kernel's uncertainty of a q tie (bf16 inputs make exact ties common), and the
    neighbouring fp16 scale of a block whose scale lies at an fp16 tie."""
    g = v.view(-1, 32)
    tg = torch.zeros_like(g) if tol is None else tol.view(-1, 32)
    amax, arg = g.abs().max(1, keepdim=True)
    dq = amax / 127
    inv = torch.where(dq > 0, 1 / dq.clamp_min(1e-300), torch.zeros_like(dq))
    t = g * inv
    q = torch.round(t)
    d16 = dq.to(torch.float16).double()
    rel = tg.gather(1, arg) / amax.clamp_min(1e-300)                 # relative uncertainty of the block maximum from the input
    # t = v / d: the norm factor cancels; what remains is the f32 rounding of v (2 roundings), d (an approximate division, 2 ulps),
    # 1/d (an approximate reciprocal, 1 ulp) and v * (1/d): at most 12 half-ulps of t
    dt = 1e-6 + 16 * U * t.abs() + inv * (tg + g.abs() * rel)
    at = t.abs()
    qtie = ((at - at.floor() - 0.5).abs() < dt).view(-1)
    step = (torch.sign(t - q) * d16).view(-1)                        # towards the other neighbour of t
    # the fp16 scale also carries the norm factor's f32 error (a sum of n squares)
    ulp = torch.exp2(torch.floor(torch.log2(dq.clamp_min(2.0 ** -14))) - 10)
    fr = dq / ulp
    stie = ((fr - fr.floor() - 0.5).abs() < fr * (rel + 8 * U + (64 * U if normed else 0)) + 1e-6)[:, 0]
    blocks, elems = stie.nonzero()[:, 0].tolist(), qtie.nonzero()[:, 0].tolist()
    alt = torch.zeros(len(blocks) + len(elems), v.numel(), dtype=v.dtype, device=v.device)
    for j, b in enumerate(blocks):
        alt[j, 32 * b:32 * b + 32] = ulp[b] * q[b]
    for j, i in enumerate(elems, len(blocks)):
        alt[j, i] = step[i]
    return (q * d16).view(-1), alt


def gemv(raw, act, bound=True, got=None, chunk=4096):
    """float64 W @ xq of the q40 rows `raw` and the q80 activation act = q80(..) and, with `bound`, the kernel's error bound of every
    row: f32 rounding of the per-block dot products (against the block scale x the block's |xq|) and of the segment / row sums
    (against sum |w x|), plus |W @ alt| for every q80 alternative. With the kernel's output `got`, the alternatives are resolved
    instead: each one moves every row at once, so the combination the kernel took is the 0/1 least-squares fit of got - W @ xq, and
    the result is W @ (xq + the chosen alternatives) with the accumulation bound alone. A fault confined to a few rows cannot be
    absorbed by such a fit."""
    xq, alt = act
    nseg = (raw.shape[1] + 31) // 32
    ax = xq.abs()
    axb = ax.view(-1, 32).sum(1)
    ys, bs, alts = [], [], []
    for r0 in range(0, raw.shape[0], chunk):
        W, S = dequant(raw[r0:r0 + chunk])
        w = W.double()
        del W
        ys.append(w @ xq)
        alts.append(w @ alt.T)
        if bound:
            w.abs_()
            bs.append(U * (nseg + 8) * (w @ ax) + 72 * U * (S.double().abs() @ axb))
        del w
    y, A = torch.cat(ys), torch.cat(alts)
    b = torch.cat(bs) if bound else None
    if A.shape[1]:
        if got is None:
            b = b + A.abs().sum(1) if bound else b
        else:
            sel = (torch.linalg.pinv(A) @ (got.double() - y)).round().clamp(0, 1)
            y = y + A @ sel
    return y, b


def gemv_rows(raw, acts, gots=None, chunk=4096):
    """gemv over the rows of a batch, every chunk of the matrix dequantised once for all of them: acts holds one q80(..) per row,
    gots (optional) the kernel's output per row. Returns one (y, bound) per row, as gemv(raw, act, got=got) computes them, except
    that where the rounded least-squares choice of up to 10 alternatives leaves the row outside its bound, the combination that
    fits best in every element is taken, and where none fits, the row keeps every alternative in its bound (gemv without `got`)."""
    X = torch.stack([xq for xq, _ in acts])
    AX = X.abs()
    AXB = AX.view(len(acts), -1, 32).sum(2)
    ALT = torch.cat([alt for _, alt in acts])
    nseg = (raw.shape[1] + 31) // 32
    ys, bs, alts = [], [], []
    for r0 in range(0, raw.shape[0], chunk):
        W, S = dequant(raw[r0:r0 + chunk])
        w = W.double()
        del W
        ys.append(w @ X.T)
        alts.append(w @ ALT.T)
        w.abs_()
        bs.append(U * (nseg + 8) * (w @ AX.T) + 72 * U * (S.double().abs() @ AXB.T))
        del w
    Y, A, B = torch.cat(ys), torch.cat(alts), torch.cat(bs)
    out, k0 = [], 0
    for i, (_, alt) in enumerate(acts):
        a, y, b = A[:, k0:k0 + alt.shape[0]], Y[:, i], B[:, i]
        k0 += alt.shape[0]
        if a.shape[1]:
            if gots is None:
                b = b + a.abs().sum(1)
            else:
                d = gots[i].double() - y
                sel = (torch.linalg.pinv(a) @ d).round().clamp(0, 1)
                if a.shape[1] <= 10 and float(((d - a @ sel).abs() / b).max()) > 1:
                    # the rounded least-squares fit can miss among a few alternatives of similar effect: try every combination
                    combos = torch.tensor([[(c >> k) & 1 for k in range(a.shape[1])] for c in range(1 << a.shape[1])],
                                          dtype=a.dtype, device=a.device)
                    worst = torch.stack([((d - a @ c).abs() / b).max() for c in combos])
                    sel = combos[int(worst.argmin())]
                    if float(worst.min()) > 1:
                        # no listed combination explains the row: keep every alternative in the bound, as gemv(got=None)
                        out.append((y, b + a.abs().sum(1)))
                        continue
                y = y + a @ sel
        out.append((y, b))
    return out


def attention(q_raw, K, V, n_pos, q_norm, rope_row, nh, eps, n_splits, bound=True):
    """float64 decode attention of the raw q [nh * hd] (QK-norm, RoPE) over rows [0, n_pos) of the bf16 caches K, V [n_kv, seq, hd],
    and its bound: f32 score error (sum |q k|), __expf error, and the f32 accumulation over the positions one warp walks."""
    nkv, _, hd = K.shape
    q = q_raw.view(nh, hd)
    if q_norm is not None:
        q = rms(q, q_norm, eps)
    q = rope(q, rope_row) / math.sqrt(hd)
    Kh = K[:, :n_pos].double().repeat_interleave(nh // nkv, 0)
    Vh = V[:, :n_pos].double().repeat_interleave(nh // nkv, 0)
    s = torch.einsum("hd,hsd->hs", q, Kh)
    pr = torch.softmax(s, -1)
    z = torch.einsum("hs,hsd->hd", pr, Vh)
    if not bound:
        return z.reshape(-1), None
    dots = torch.einsum("hd,hsd->hs", q.abs(), Kh.abs())
    span = (s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True))
    eps_s = U * (16 * dots + 8 + 4 * (s.amax(-1, keepdim=True) - s + span))
    eff = max(1, min(n_splits, (n_pos + 255) // 256))
    depth = math.ceil(math.ceil(n_pos / eff) / 16) + 16 + eff + 8
    b = torch.einsum("hs,hsd->hd", pr * eps_s, (Vh - z[:, None, :]).abs()) + U * depth * torch.einsum("hs,hsd->hd", pr, Vh.abs())
    return z.reshape(-1), b.reshape(-1) + U * z.abs().reshape(-1)


def bf16_ulp(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def worst(got, want, bound):
    r = (got.double() - want).abs() / bound
    return float(torch.nan_to_num(r, nan=float("inf")).max())


def kv_rows(R, L, qkv, rope_row):
    """float64 K row (QK-norm + RoPE of the raw k) and the V row of the raw q|k|v, [n_kv, hd] each."""
    k = qkv[R.q_dim:R.q_dim + R.kv_dim].view(R.nkv, R.hd)
    if L["k_norm"] is not None:
        k = rms(k, L["k_norm"], R.eps)
    return rope(k, rope_row), qkv[R.q_dim + R.kv_dim:].view(R.nkv, R.hd)


# ---- engine-level stage checks (test_gpu_prefill_chain.py, test_gpu_batched_steps.py) -----------------------------------------
def rope_rows(x, rows):
    """x [T, H, hd] rotated per token by rows [T, hd/2, 2]."""
    a, b = x[..., 0::2], x[..., 1::2]
    c, s = rows[:, None, :, 0], rows[:, None, :, 1]
    out = torch.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = a * s + b * c
    return out


def norm_rope(y, b, w, rows, eps):
    """QK-norm (w, or None) and RoPE of y [T, H, hd] with error bound b, returning (value, bound): the norm carries b through its
    derivative plus 2^-18 relative for the f32 norm; a rotated pair takes the bounds of both inputs plus 4 f32 roundings."""
    hd = y.shape[-1]
    if w is not None:
        ms = (y * y).mean(-1, keepdim=True) + eps
        yn = w * y / ms.sqrt()
        b = w.abs() / ms.sqrt() * (b + y.abs() * (y.abs() * b).sum(-1, keepdim=True) / (hd * ms)) + REL_NORM * yn.abs()
        y = yn
    pair = b[..., 0::2] + b[..., 1::2] + 4 * U * (y[..., 0::2].abs() + y[..., 1::2].abs())
    return rope_rows(y, rows), pair.repeat_interleave(2, -1)



def ratio(got, want, bound):
    r = (got.double() - want).abs() / bound
    return float(torch.nan_to_num(r, nan=float("inf")).max())



def k_rows_ok(got_k, k, kn):
    """K rows against bf16 of the f64 rotation k of the normalised raw k `kn`: within 1 bf16 ulp plus the f32 rounding of the
    rotation (4 roundings of the pair's magnitude, which cancellation can make exceed an ulp of the result) and, with QK-norm,
    2^-18 of it; at most 1 in 64 off the nearest. Returns (worst error / bound, count ok)."""
    kb = k.to(torch.bfloat16).double()
    off = (got_k.double() - kb).abs()
    pair = (kn[..., 0::2].abs() + kn[..., 1::2].abs()).repeat_interleave(2, -1)
    worst_r = float((off / (bf16_ulp(kb) + (4 * U + REL_NORM) * pair)).max())
    n_off = int((off != 0).sum())
    return worst_r, n_off <= max(4, k.numel() // 64)



def _random_caches(eng, seed):
    """Random starting caches in the engine's storage: bf16 N(0, 1), or q80 ints in [-127, 127] with f16 scales of 0.005 .. 0.015
    (values of about the same spread) as (K values, V values, K scales, V scales)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if eng.kv_cache_float_type == "bf16":
        return ([torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.k_cache],
                [torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.v_cache])
    vals = [torch.randint(-127, 128, c.shape, generator=g, device="cuda", dtype=torch.int8) for c in eng.k_cache + eng.v_cache]
    scales = [(torch.rand(s.shape, generator=g, device="cuda") * 0.01 + 0.005).half() for s in eng.k_scale + eng.v_scale]
    n = len(eng.k_cache)
    return vals[:n], vals[n:], scales[:n], scales[n:]


def _scale_rows(eng, s):
    """A q80 scale plane as [nKv, seq, hd / 32] (without its tail padding)."""
    nkv, seq, hd = eng.k_cache[0].shape
    return s[:nkv * seq * hd // 32].view(nkv, seq, hd // 32)


def _load(eng, caches, poison_from=None):
    """Copies the caches in; from row poison_from on, bf16 values or q80 scales hold NaN."""
    q8 = eng.kv_cache_float_type == "q80"
    for d, s in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
        d.copy_(s)
        if poison_from is not None and not q8:
            d[:, poison_from:] = float("nan")
    if q8:
        for d, s in zip(eng.k_scale + eng.v_scale, caches[2] + caches[3]):
            d.copy_(s)
            if poison_from is not None:
                _scale_rows(eng, d)[:, poison_from:] = float("nan")



def attn_operands(eng, tc):
    """Layer 0's K and V as the attention kernels multiply them: the bf16 cache as stored; q80: the tensor-core tiles widened to
    bf16(f32(int8) x f32(f16 scale)), or the exact dequantisation the CUDA-core kernels use (f64)."""
    if eng.kv_cache_float_type == "bf16":
        return eng.k_cache[0], eng.v_cache[0]
    out = []
    for vals, sc in ((eng.k_cache[0], eng.k_scale[0]), (eng.v_cache[0], eng.v_scale[0])):
        nkv, seq, hd = vals.shape
        x = vals.float().view(nkv, seq, hd // 32, 32) * _scale_rows(eng, sc).float()[..., None]
        out.append(x.view(nkv, seq, hd).bfloat16() if tc else x.view(nkv, seq, hd).double())
    return out


def check_kv_rows(eng, st, tag, p, k, kn, v):
    """The K/V rows layer 0 stored at p .. p + T - 1 against the f64 K rows k (the rotation of the normalised raw k `kn`) and the
    raw V rows v, each [T, nKv, hd]. bf16: k_rows_ok, V exactly bf16(v). q80: every 32-block's f16 scale within one f16 step of
    f16(amax / 127), every int within 0.5 of x / (amax / 127), plus 1e-3 and, for K, the f32 rounding of the rotation in units
    of the scale; the ratio is the worst int distance over that bound."""
    T = k.shape[0]
    if eng.kv_cache_float_type == "bf16":
        Kc, Vc = eng.k_cache[0], eng.v_cache[0]
        r, ok = k_rows_ok(Kc[:, p:p + T].transpose(0, 1), k, kn)
        assert ok, f"{tag} p={p}: K rows off the nearest bf16 too often"
        st.r(f"{tag} k rows", r)
        assert torch.equal(Vc[:, p:p + T].transpose(0, 1), v.float().to(torch.bfloat16)), f"{tag} p={p}: V rows are not bf16(v)"
        return
    pair = (kn[..., 0::2].abs() + kn[..., 1::2].abs()).repeat_interleave(2, -1)
    for name, x, err, vals, sc in (("k", k, (4 * U + REL_NORM) * pair, eng.k_cache[0], eng.k_scale[0]),
                                   ("v", v, torch.zeros_like(v), eng.v_cache[0], eng.v_scale[0])):
        xb = x.reshape(T, -1, 32)
        d = xb.abs().amax(-1, keepdim=True) / 127
        got_s = _scale_rows(eng, sc)[:, p:p + T].transpose(0, 1).reshape(T, -1, 1).double()
        want_s = d.half().double()
        st.r(f"{tag} q80 {name} scales", ratio(got_s, want_s, want_s * 2.0 ** -10 + 1e-30))
        q = vals[:, p:p + T].transpose(0, 1).reshape(T, -1, 32).double()
        t = torch.where(d > 0, xb / d.clamp_min(1e-300), torch.zeros_like(xb))
        slack = 1e-3 + torch.where(d > 0, err.reshape(T, -1, 32) / d.clamp_min(1e-300), torch.zeros_like(xb))
        st.r(f"{tag} q80 {name} ints", ratio(q, t, 0.5 + slack))



class Stats:
    def __init__(self):
        self.ratios, self.controls = {}, {}

    def r(self, k, v):
        self.ratios[k] = max(self.ratios.get(k, 0.0), v)

    def c(self, k, v):
        """A negative control counts where it lands furthest: the check fails by that factor if the kernel has that fault."""
        self.controls[k] = max(self.controls.get(k, 0.0), v)

    def report(self, tag):
        print(f"\n[{tag}] worst error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in self.ratios.items()))
        if self.controls:
            print(f"[{tag}] negative control / bound: " + ", ".join(f"{k} {v:.0f}" for k, v in self.controls.items()))
        for k, v in self.ratios.items():
            assert v <= 1.0, f"{tag}: {k} exceeds its bound ({v:.3f})"
        for k, v in self.controls.items():
            assert v >= CONTROL_MIN, f"{tag}: the negative control '{k}' is only {v:.1f}x its bound"
