"""Float64 reference helpers shared by the q40 matrix tests (tests/test_gpu_gemm_tc.py, tests/test_gpu_moe.py, tests/test_gpu_gemv.py).

* Random q40 matrices as raw 18-byte blocks (f16 scale + 16 bytes of nibbles) and their device layout.
* The weights the tensor-core dequant warps build from them: rn_bf16(rn_bf16(f16 scale) * (q - 8)).
* The q80 grid of decode activations, with the ambiguity of a rounding whose input is only known within an interval.
* Checks of a kernel's values against a float64 reference with a per-element bound, or against the bf16 roundings of the two ends
  of an interval.
"""
import math
import zlib

import torch


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

    def _parts(self, e):
        blk = self.n // 32
        return q40_parts(self.raw[e * self.rows * blk:(e + 1) * self.rows * blk], self.rows, self.n)

    def w_exact(self, e):
        """Matrix e dequantised exactly (the decode GEMV's weights), f64 [rows][n], and |w| + 8 |scale| (its f32 error scale)."""
        sc, q = self._parts(e)
        s = sc.double().repeat_interleave(32, dim=1)
        return s * q, s.abs() * (q.abs() + 8)

    def w_tc(self, e=0):
        """Matrix e as the tensor-core dequant builds it."""
        return w_tc_of(*self._parts(e))


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
