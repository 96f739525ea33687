"""Decode GEMVs against float64: gemvQ40Kernel ("ldg", per-thread loads, gemv_q40.cu), gemvQ40TmaKernel ("tma", TMA ring,
gemv_q40_tma.cu) with its fused arg-max epilogue, argmaxAdvanceKernel (decode_ops.cu) and gemvDenseKernel (f32 / f16 weights,
gemv_dense.cu).

Every q40 case asserts the plan it runs through dl_gemv_q40_plan (kernel, ring geometry, launches the batch is split into), so a
change of the dispatch moves no case off its path silently. The plan table pins the plans of the production shapes at 132 and
114 SMs; it launches nothing and runs without a GPU.

Reference: float64 over exactly what the kernels multiply. A q40 weight is f16 scale * (nibble - 8), exact in float64. The
activations are the q80 grid of the (rmsnorm'd) input: d = f16(amax / 127), q = rint(x / d) per block of 32 (q40_ref.q80_ref).
The kernel's own input to that rounding differs from the float64 one by fast division and reciprocal (2^-20 relative), or by the
f32 rmsnorm (fast rsqrt, f32 sum of squares, 2^-18 relative). q80_ref rounds both ends of that interval, and where they differ
the bound gains the distance between them. Bounds per output element, with S = sum over the dot product of |a| * (|w| + 8 |scale|):
the kernel multiplies unsigned nibbles and subtracts 8 * scale * sum(q) afterwards, so its running values scale with |w| + 8 |scale|.
* q40 f32 accumulation: 2^-18 * S. Per 32-block the kernel rounds three times: dx * dot, dx8 = f16(d) * 8 * sum(q) is exact, then
  the difference, then the product with the weight scale. A 32-block warp sum adds five roundings (the TMA kernel's transposing
  butterfly also five), and the segment sum one per segment (<= 28 at the shapes here). That is under 40 roundings of values at
  most S, each <= 2^-24 S: 2^-18.7 S. 2^-18 S is 64 of them.
* Residual add: 2^-22 of |x0| + |result|. SiLU (__expf, fast division): 2^-19 relative. tanh-GELU: 2^-20 (|gelu(g)| + |g|).
  The bound on gate and up carries through |silu'| <= 1.1 and |gelu'| <= 1.13.
* Dense GEMV: a lane runs one fmaf chain over n / 32 weights (the unrolled chunks of a lane are consecutive in that chain), then a
  5-level warp sum: (n / 32 + 6) * 2^-24 * S with S = |x| @ |w|. The rmsnorm'd activations add 2^-18 * S.

Exactness (the decode counterpart of the one-hot GEMM rows): token t has one non-zero 32-block b_t with values k_i * s rounded to
f32, k_i integers in [-127, 127] with one of them +-127, s = h (1 + j 2^-14), h an f16 value and j in +-{1, 2, 3}. Then
f16(amax / 127) = h with a wide margin, q = k_i although the kernel divides approximately, and every other block quantises to exact
zeros. So out[t, r] = dw[r, b_t] * h * sum_i k_i (nib_i - 8) within the three f32 roundings of the block's product; with
power-of-two weight scales and h, bitwise. PRO_RMSNORM: x = +-2^c everywhere and eps = 0 (the mean square is exact), the norm
weight carries k_i * s in the hot block and zeros elsewhere. That pins the nibble and plane order, dx8, the f16 rounding of the
activation scale, rows, tiles, ring stages, token planes and a partial last segment (n = 18560: 19 segments, the last of 4 blocks).

On an H100 80GB HBM3 (132 SMs, 700 W power limit) the file runs in about 12 s. The largest error / bound is 0.54 on both q40
kernels and 0.035 on the dense one; every block-hot case with power-of-two scales is bitwise exact.

The split: when neither q40 kernel holds nb tokens in shared memory (Qwen3-14B and Llama-3.3-70B logits, Llama-3.3-70B W2, all at
8 tokens on one GPU), the batch runs as launches of nb / 2 tokens. Those shapes returned -2 before; test_plan_table and
test_production_shapes run them.
"""
import math

import pytest
import torch

from q40_ref import assert_within, gen, q40_parts, q80_ref

C_ACC = 2.0 ** -18
C_SUM = 2.0 ** -22
C_SILU = 2.0 ** -19
C_GELU = 2.0 ** -20
C_HOT = 2.0 ** -22     # block-hot outputs: three f32 roundings
REL_NORM = 2.0 ** -18
REL_PLAIN = 2.0 ** -20
SILU, GELU = 0, 1
NAN_F32 = 0x7FC0DEAD
EPS = 1e-5

STORE, RESID, SWIGLU = 0, 1, 2
RMS, PLAIN = 0, 1
# instantiated (pro, epi) -> batch widths, both q40 kernels and the dense one (PLAIN / SWIGLU: q40 only, one token)
COMBOS = {(RMS, STORE): (1, 2, 4, 8), (PLAIN, RESID): (1, 2, 4, 8), (RMS, SWIGLU): (1, 2, 4, 8), (PLAIN, STORE): (1, 2, 4, 8),
          (PLAIN, SWIGLU): (1,)}
INSTANCES = [(p, e, nb) for (p, e), nbs in COMBOS.items() for nb in nbs]


def _ops():
    from distributed_llama_b200 import ops
    return ops


def _device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- plan table (no GPU) -------------------------------------------------------------------------------------------------
MODELS = {
    "llama-3.1-8b": dict(qkv=(6144, 4096), wo=(4096, 4096), w13=(28672, 4096), w2=(4096, 14336), logits=(128256, 4096)),
    "qwen3-0.6b": dict(qkv=(4096, 1024), wo=(1024, 2048), w13=(6144, 1024), w2=(1024, 3072), logits=(151936, 1024)),
    "qwen3-8b": dict(qkv=(6144, 4096), wo=(4096, 4096), w13=(24576, 4096), w2=(4096, 12288), logits=(151936, 4096)),
    "qwen3-14b": dict(qkv=(7168, 5120), wo=(5120, 5120), w13=(34816, 5120), w2=(5120, 17408), logits=(151936, 5120)),
    "llama-3.3-70b": dict(qkv=(10240, 8192), wo=(8192, 8192), w13=(57344, 8192), w2=(8192, 28672), logits=(128256, 8192)),
    # one rank's slices under tensor parallelism: WO and W2 carry the in-kernel all-reduce, which only the TMA kernel has
    "llama-3.3-70b-tp2": dict(qkv=(5120, 8192), wo=(8192, 4096), w13=(28672, 8192), w2=(8192, 14336), logits=(64128, 8192)),
    "llama-3.3-70b-tp8": dict(qkv=(1280, 8192), wo=(8192, 1024), w13=(7168, 8192), w2=(8192, 3584), logits=(16032, 8192)),
    "llama-3.1-8b-slice8": dict(qkv=(768, 4096), wo=(4096, 512), w13=(3584, 4096), w2=(4096, 1792), logits=(16032, 4096)),
}
TP = {"llama-3.3-70b-tp2", "llama-3.3-70b-tp8", "llama-3.1-8b-slice8"}
MATRIX = {"qkv": (RMS, STORE), "wo": (PLAIN, RESID), "w13": (RMS, SWIGLU), "w2": (PLAIN, RESID), "logits": (RMS, STORE)}
NBS = (1, 2, 4, 8)
# "kernel/stageRows/nStages/smemBytes" per nb in NBS, "xL": the batch runs as L launches. kernel 1 = ldg, 2 = tma.
PLAN_TABLE = {
    132: {
        "llama-3.1-8b": {"qkv": "2/16/2/80288 2/16/3/123072 2/16/3/134912 2/16/3/158592", "wo": "2/16/2/80032 2/16/2/85696 2/16/2/97024 2/16/2/119680", "w13": "2/16/2/83008 2/16/5/202240 2/16/5/219520 2/16/4/217216", "w2": "2/4/2/84976 2/4/5/201568 2/4/4/208960 2/4/2/223744", "logits": "2/16/2/95072 2/16/5/226368 2/16/4/230912 2/16/1/203136"},
        "qwen3-0.6b": {"qkv": "2/64/1/38920 2/64/1/40336 2/64/1/43168 2/64/1/48832", "wo": "2/32/1/40144 2/32/1/42784 2/32/1/48064 2/32/1/58624", "w13": "2/64/1/38984 2/64/1/40464 2/64/1/43424 2/64/1/49344", "w2": "2/20/1/39160 2/20/1/43120 2/20/1/51040 2/20/1/66880", "logits": "2/64/2/80264 2/64/5/196752 2/64/5/208544 2/64/4/195264"},
        "qwen3-8b": {"qkv": "2/16/2/80288 2/16/3/123072 2/16/3/134912 2/16/3/158592", "wo": "2/16/2/80032 2/16/2/85696 2/16/2/97024 2/16/2/119680", "w13": "2/16/2/82528 2/16/5/201280 2/16/5/217600 2/16/4/213376", "w2": "2/4/3/100576 2/4/7/228160 2/4/5/206848 2/4/3/219520", "logits": "2/16/2/97952 2/16/4/195264 2/16/3/205568 2/16/1/226176"},
        "qwen3-14b": {"qkv": "2/12/3/111880 2/12/5/188560 2/12/5/203680 2/12/4/199360", "wo": "2/12/3/111560 2/12/4/153360 2/12/4/167840 2/12/4/196800", "w13": "2/12/2/81480 2/12/5/196880 2/12/5/220320 2/12/3/198080", "w2": "2/4/2/103592 2/4/4/206544 2/4/3/216608 1/0/0/195920", "logits": "2/12/2/99240 2/12/4/197840 2/12/3/222240 2/12/3/222240x2"},
        "llama-3.3-70b": {"qkv": "2/8/2/87168 2/8/5/210560 2/8/4/199296 2/8/3/213632", "wo": "2/8/2/86720 2/8/5/209664 2/8/4/197504 2/8/3/210048", "w13": "2/8/2/98624 2/8/4/196608 2/8/3/208256 1/0/0/193616", "w2": "1/0/0/43088 1/0/0/86096 1/0/0/172112 1/0/0/172112x2", "logits": "2/8/1/78912 2/8/4/230912 2/8/1/203136 2/8/1/203136x2"},
        "llama-3.3-70b-tp2": {"qkv": "2/8/2/85952 2/8/5/208128 2/8/5/231296 2/8/3/203904", "wo": "2/16/2/80544 2/16/4/160448 2/16/4/172800 2/16/4/197504", "w13": "2/8/2/91648 2/8/5/219520 2/8/4/217216 2/8/2/212608", "w2": "2/4/2/86768 2/4/5/205152 2/4/4/216128 2/4/1/205824", "logits": "2/8/2/100224 2/8/4/199808 2/8/3/214656 1/0/0/206416"},
        "llama-3.3-70b-tp8": {"qkv": "2/8/2/84992 2/8/2/95616 2/8/2/116864 2/8/2/159360", "wo": "2/64/1/39048 2/64/1/40592 2/64/1/43680 2/64/1/49856", "w13": "2/8/2/86464 2/8/5/209152 2/8/4/196480 2/8/3/208000", "w2": "2/16/3/102944 2/16/4/140736 2/16/4/151808 2/16/4/173952", "logits": "2/8/2/88576 2/8/5/213376 2/8/4/204928 2/8/3/224896"},
        "llama-3.1-8b-slice8": {"qkv": "2/16/1/42752 2/16/1/48000 2/16/1/58496 2/16/1/79488", "wo": "2/64/1/19848 2/64/1/20624 2/64/1/22176 2/64/1/25280", "w13": "2/16/2/79968 2/16/2/85568 2/16/2/96768 2/16/2/119168", "w2": "2/32/1/35408 2/32/1/37920 2/32/1/42944 2/32/1/52992", "logits": "2/16/2/81472 2/16/5/199168 2/16/5/213376 2/16/4/204928"},
    },
    114: {
        "llama-3.1-8b": {"qkv": "2/16/2/80384 2/16/4/160128 2/16/4/172160 2/16/4/196224", "wo": "2/16/2/80096 2/16/3/122688 2/16/3/134144 2/16/3/157056", "w13": "2/16/2/83552 2/16/5/203328 2/16/5/221696 2/16/4/221568", "w2": "2/4/2/85200 2/4/5/202016 2/4/4/209856 2/4/2/225536", "logits": "2/16/2/97536 2/16/5/231296 2/16/3/203904 2/16/1/222848"},
        "qwen3-0.6b": {"qkv": "2/64/1/38936 2/64/1/40368 2/64/1/43232 2/64/1/48960", "wo": "2/32/1/40160 2/32/1/42816 2/32/1/48128 2/32/1/58752", "w13": "2/64/1/39008 2/64/1/40512 2/64/1/43520 2/64/1/49536", "w2": "2/20/1/39184 2/20/1/43168 2/20/1/51136 2/20/1/67072", "logits": "2/64/2/80992 2/64/5/198208 2/64/5/211456 2/64/4/201088"},
        "qwen3-8b": {"qkv": "2/16/2/80384 2/16/4/160128 2/16/4/172160 2/16/4/196224", "wo": "2/16/2/80096 2/16/3/122688 2/16/3/134144 2/16/3/157056", "w13": "2/16/2/82976 2/16/5/202176 2/16/5/219392 2/16/4/216960", "w2": "2/4/3/100768 2/4/7/228544 2/4/5/207616 2/4/3/221056", "logits": "2/16/2/100864 2/16/4/201088 2/16/3/217216 1/0/0/211792"},
        "qwen3-14b": {"qkv": "2/12/3/112040 2/12/6/223440 2/12/5/204320 2/12/4/200640", "wo": "2/12/3/111680 2/12/4/153600 2/12/4/168320 2/12/4/197760", "w13": "2/12/2/82320 2/12/5/198560 2/12/5/223680 2/12/3/204800", "w2": "2/4/2/104000 2/4/4/207360 2/4/3/218240 1/0/0/199184", "logits": "2/12/2/102880 2/12/4/205120 2/12/2/202240 2/12/2/202240x2"},
        "llama-3.3-70b": {"qkv": "2/8/2/87552 2/8/5/211328 2/8/4/200832 2/8/3/216704", "wo": "2/8/2/86976 2/8/5/210176 2/8/4/198528 2/8/3/212096", "w13": "2/8/2/100800 2/8/4/200960 2/8/3/216960 1/0/0/211024", "w2": "1/0/0/43984 1/0/0/87888 1/0/0/175696 1/0/0/175696x2", "logits": "2/8/1/83840 2/8/3/203904 2/8/1/222848 2/8/1/222848x2"},
        "llama-3.3-70b-tp2": {"qkv": "2/8/2/86144 2/8/5/208512 2/8/4/195200 2/8/3/205440", "wo": "2/16/2/80672 2/16/5/197568 2/16/5/210176 2/16/4/198528", "w13": "2/8/2/92736 2/8/5/221696 2/8/4/221568 2/8/2/221312", "w2": "2/4/2/87216 2/4/5/206048 2/4/4/217920 2/4/1/209408", "logits": "2/8/2/102720 2/8/4/204800 2/8/3/224640 1/0/0/226384"},
        "llama-3.3-70b-tp8": {"qkv": "2/8/2/85056 2/8/2/95744 2/8/2/117120 2/8/2/159872", "wo": "2/64/2/75944 2/64/2/77520 2/64/2/80672 2/64/2/86976", "w13": "2/8/2/86720 2/8/5/209664 2/8/4/197504 2/8/3/210048", "w2": "2/16/3/103072 2/16/5/173248 2/16/5/184576 2/16/5/207232", "logits": "2/8/2/89216 2/8/5/214656 2/8/4/207488 2/8/3/230016"},
        "llama-3.1-8b-slice8": {"qkv": "2/16/1/42784 2/16/1/48064 2/16/1/58624 2/16/1/79744", "wo": "2/64/1/19864 2/64/1/20656 2/64/1/22240 2/64/1/25408", "w13": "2/16/2/80032 2/16/2/85696 2/16/2/97024 2/16/2/119680", "w2": "2/32/2/67696 2/32/2/70240 2/32/2/75328 2/32/2/85504", "logits": "2/16/2/81792 2/16/5/199808 2/16/5/214656 2/16/4/207488"},
    },
}
# no kernel holds 8 tokens of these on one GPU: the batch runs as two launches of 4 (these returned -2 before the split)
SPLIT_ROWS = [("qwen3-14b", "logits"), ("llama-3.3-70b", "logits"), ("llama-3.3-70b", "w2")]


def _impl(model, mat):
    return "tma" if model in TP and mat in ("wo", "w2") else "auto"


def _fmt(p):
    return f"{p.kernel}/{p.stage_rows}/{p.n_stages}/{p.smem_bytes}" + (f"x{p.launches}" if p.launches > 1 else "")


def plan_of(pro, epi, nb, d, n, sms, impl="auto"):
    return _ops().gemv_q40_plan(pro, epi, nb, d, n, num_sms=sms, impl=impl)


@pytest.mark.parametrize("sms", [132, 114])
def test_plan_table(sms):
    """QKV, WO, W1|W3, W2 and logits of the production models at nb 1, 2, 4, 8 (H100 SXM: 132 SMs, PCIe: 114): every plan
    launches, grid and tile rows follow the pair split, and each matches the pinned row."""
    for model, mats in MODELS.items():
        for mat, (d, n) in mats.items():
            got = []
            for nb in NBS:
                p = plan_of(*MATRIX[mat], nb, d, n, sms, _impl(model, mat))
                assert p.rc == 0, (model, mat, nb, p)
                pairs = d // 2
                assert p.grid == min(pairs, sms) and p.max_tile_rows == 2 * -(-pairs // p.grid), p
                assert p.smem_bytes <= 227 * 1024 and (p.kernel == 1) == (p.stage_rows == 0), p
                got.append(_fmt(p))
            assert " ".join(got) == PLAN_TABLE[sms][model][mat], f"{model} {mat} at {sms} SMs: {' '.join(got)}"
    for model, mat in SPLIT_ROWS:
        d, n = MODELS[model][mat]
        assert plan_of(*MATRIX[mat], 8, d, n, sms).launches == 2
        assert plan_of(*MATRIX[mat], 8, d, n, sms, "ldg").launches == 2


def test_plan_edges():
    """The TMA kernel needs n % 128 == 0 (rc 1, auto takes the fallback); odd d and n % 32 != 0 are refused; combinations
    that are not compiled are refused (-3) instead of launched; a split never applies to the arg-max epilogue."""
    assert plan_of(RMS, STORE, 1, 1000, 4160, 132, "tma").rc == 1
    p = plan_of(RMS, STORE, 1, 1000, 4160, 132)
    assert p.rc == 0 and p.kernel == 1 and p.launches == 1
    assert plan_of(RMS, STORE, 1, 1001, 4096, 132).rc == -1
    assert plan_of(RMS, STORE, 1, 1000, 4112, 132).rc == -1
    assert plan_of(PLAIN, SWIGLU, 2, 1000, 4096, 132).rc == -3
    assert plan_of(RMS, 3, 2, 1000, 4096, 132).rc == -3
    assert plan_of(RMS, 3, 1, 1000, 4096, 132, "tma").rc == 0
    d, n = MODELS["llama-3.3-70b"]["w2"]
    assert plan_of(RMS, 3, 8, d, n, 132).rc == -2


def test_dense_batch_cap_fits():
    """Dense weight files: the engine's batch cap (runtime.engine.dense_max_batch) keeps every matrix of every dense preset that
    it accepts within the dense GEMV's shared memory at that batch width."""
    from distributed_llama_b200.models.config import PRESETS
    from distributed_llama_b200.runtime.engine import dense_max_batch
    ops = _ops()
    checked = 0
    for name, c in PRESETS.items():
        if c.n_experts:
            continue                      # the MoE engine runs one token per launch
        hd = c.head_dim or c.dim // c.n_heads
        q, kv = c.n_heads * hd, c.n_kv_heads * hd
        try:
            nb = dense_max_batch(8, c.dim, c.hidden_dim, q)
        except ValueError:
            continue
        mats = [(q + 2 * kv, c.dim), (c.dim, q), (2 * c.hidden_dim, c.dim), (c.dim, c.hidden_dim), (c.vocab_size, c.dim)]
        for sms in (132, 114):
            for d, n in mats:
                assert ops.gemv_dense_smem_bytes(d, n, nb, sms) <= 227 * 1024, (name, d, n, nb, sms)
        checked += 1
    assert checked >= 8


# ---- helpers -------------------------------------------------------------------------------------------------------------
class Q40:
    """Random q40 matrix [d][n]: raw 18-byte blocks on the device, the device layout, and float64 views by row range.
    scales: "f16" random +-(0.5 .. 1.5) / (4 sqrt(n)); "pow2" +-2^-e with e in 5..9."""

    def __init__(self, d, n, seed=0, scales="f16"):
        g = gen("gemv-q40", d, n, seed, scales)
        nb = d * n // 32
        if scales == "pow2":
            sc = torch.exp2(-torch.randint(5, 10, (nb,), device="cuda", generator=g).float())
        else:
            sc = (torch.rand(nb, device="cuda", generator=g) + 0.5) / (4.0 * math.sqrt(n))
        sc = torch.where(torch.rand(nb, device="cuda", generator=g) < 0.5, -sc, sc).half()
        self.raw = torch.empty(nb, 18, dtype=torch.uint8, device="cuda")
        self.raw[:, :2] = sc.view(torch.uint8).view(nb, 2)
        self.raw[:, 2:] = torch.randint(0, 256, (nb, 16), dtype=torch.uint8, device="cuda", generator=g)
        self.d, self.n = d, n
        self._dev = None

    def device(self):
        if self._dev is None:
            ops = _ops()
            self._dev = ops.DeviceQ40.empty(self.d, self.n)
            ops.repack_q40(self.raw.reshape(-1), self.d, self.n, self._dev)
        return self._dev

    def parts(self, r0, r1):
        blk = self.n // 32
        return q40_parts(self.raw[r0 * blk:r1 * blk], r1 - r0, self.n)

    def chunks(self):
        """(r0, r1, w f64 [r1 - r0][n], |w| + 8 |scale|) over row chunks of at most 2^26 elements."""
        step = max(2, (1 << 26) // self.n // 2 * 2)
        for r0 in range(0, self.d, step):
            r1 = min(self.d, r0 + step)
            sc, q = self.parts(r0, r1)
            s = sc.double().repeat_interleave(32, dim=1)
            yield r0, r1, s * q, s.abs() * (q.abs() + 8)


def rms64(x, w, eps):
    x = x.double()
    return w.double() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def gemv_ref(W, a, amb):
    """a @ w^T and its accumulation + q80-ambiguity bound, by row chunks."""
    ref = torch.empty(a.shape[0], W.d, dtype=torch.float64, device="cuda")
    tol = torch.empty_like(ref)
    for r0, r1, w, s in W.chunks():
        ref[:, r0:r1] = a @ w.T
        tol[:, r0:r1] = C_ACC * (a.abs() @ s.T) + amb @ w.abs().T
    return ref, tol


def glu_ref(gu, e_gu, act_fn):
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


def inputs(nb, n, d, seed):
    g = gen("gemv-in", nb, n, d, seed)
    x = torch.randn(nb, n, device="cuda", generator=g) * 2.0
    nw = 1.0 + 0.1 * torch.randn(n, device="cuda", generator=g)
    x0 = torch.randn(nb, d, device="cuda", generator=g)
    return x, nw, x0


def out_cols(epi, d):
    return d // 2 if epi == SWIGLU else d


def run_q40(W, x, pro, epi, *, nw=None, x0=None, impl="auto", sms=0, act_fn=SILU, eps=EPS, out=None):
    nb = x.shape[0]
    if out is None:
        out = x0[:nb].clone() if epi == RESID else torch.full((nb, out_cols(epi, W.d)), float("nan"), device="cuda")
    _ops().gemv_q40(W.device(), x, pro=pro, epi=epi, out=out, norm_w=nw, eps=eps, num_sms=sms or _device_sms(), impl=impl,
                    act_fn=act_fn)
    torch.cuda.synchronize()
    return out


RATIOS = {}


def check_q40(W, x, pro, epi, got, *, nw=None, x0=None, act_fn=SILU, eps=EPS, what=""):
    """got against float64 from the q80 grid of the (rmsnorm'd) input; returns the largest error / bound."""
    y, rel = (rms64(x, nw, eps), REL_NORM) if pro == RMS else (x.double(), REL_PLAIN)
    a, amb = q80_ref(y, rel)
    ref, tol = gemv_ref(W, a, amb)
    if epi == STORE:
        return assert_within(got, ref, tol, what)
    if epi == RESID:
        r = x0[:x.shape[0]].double() + ref
        return assert_within(got, r, tol + C_SUM * (x0[:x.shape[0]].double().abs() + r.abs()), what)
    h, eh = glu_ref(ref, tol, act_fn)
    return assert_within(got, h, eh, what)


def assert_plan(pro, epi, nb, d, n, sms, impl, kernel, launches=1):
    p = plan_of(pro, epi, nb, d, n, sms, impl)
    assert p.rc == 0 and p.kernel == kernel and p.launches == launches, f"{d}x{n} nb={nb} {impl} at {sms} SMs: {p}"
    return p


# ---- block-hot exactness -------------------------------------------------------------------------------------------------
# 500 row pairs over the SMs: uneven tiles. n = 18560: 580 blocks, 18 full segments + 4 blocks; n = 2176: 68 blocks, 2 + 4.
HOT_D, HOT_N = 1000, (18560, 2176)
# the TMA kernel cannot hold 8 token planes of 580 blocks next to its ring (auto takes the per-thread-load kernel there)
TMA_REFUSES = {("tma", 18560, 8)}


def hot_inputs(nb, n, rnd, pro, pow2, seed):
    """Per token: the hot block, its 32 integers k (signs of x folded in), the f16 scale h, and (x, norm weight) carrying k * s."""
    g = torch.Generator().manual_seed(seed * 1000 + rnd * 10 + nb)
    nblk = n // 32
    spots = [0, nblk // 2, nblk - 1]                         # first, middle and last (partial) segment
    x = torch.zeros(nb, n)
    nw = torch.zeros(n)
    blocks, ks, hs = [], [], []
    for t in range(nb):
        step = (t // 3) * (1 if (t + rnd) % 3 == 0 else -1)
        b = spots[(t + rnd) % 3] + step
        k = torch.randint(-127, 128, (32,), generator=g)
        k[int(torch.randint(0, 32, (1,), generator=g))] = 127 if torch.rand(1, generator=g).item() < 0.5 else -127
        if pow2:
            h = 2.0 ** -int(torch.randint(3, 8, (1,), generator=g))
        else:
            h = torch.tensor(0.01 + 0.05 * torch.rand(1, generator=g).item()).half().double().item()
        j = [-3, -2, -1, 1, 2, 3][int(torch.randint(0, 6, (1,), generator=g))]
        v = (k.double() * (h * (1.0 + j * 2.0 ** -14))).float()
        if pro == RMS:
            # x = +-2^c everywhere, eps = 0: rmsnorm(x) = sign(x) * normW. The norm weight is shared by the tokens, so they
            # all use token 0's hot block and k, each with the signs of its own x
            c = int(torch.randint(-3, 4, (1,), generator=g))
            sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
            x[t] = sign * 2.0 ** c
            if t == 0:
                nw[32 * b:32 * b + 32] = v
                k0, b0, h0 = k, b, h
            blocks.append(b0), hs.append(h0), ks.append(k0 * sign[32 * b0:32 * b0 + 32].long())
        else:
            x[t, 32 * b:32 * b + 32] = v
            blocks.append(b), ks.append(k), hs.append(h)
    return x.cuda(), nw.cuda(), blocks, ks, hs


def hot_ref(W, blocks, ks, hs):
    """float64 out[t, r] = dw[r, b_t] * h_t * sum_i k_i (nib_i - 8) and the bound of its three f32 roundings."""
    sc, q = W.parts(0, W.d)
    ref, tol = [], []
    for b, k, h in zip(blocks, ks, hs):
        kd = k.double().cuda()
        qb = q[:, 32 * b:32 * b + 32]
        dw = sc[:, b].double()
        ref.append(dw * h * (qb @ kd))
        tol.append(C_HOT * dw.abs() * h * ((qb + 8) @ kd.abs() + 8 * kd.sum().abs()))
    return torch.stack(ref), torch.stack(tol)


HOT_W = {}


def hot_matrix(n, scales):
    if (n, scales) not in HOT_W:
        HOT_W[n, scales] = Q40(HOT_D, n, 5, scales)
    return HOT_W[n, scales]


@pytest.mark.gpu
@pytest.mark.parametrize("scales", ["pow2", "f16"])
@pytest.mark.parametrize("impl", ["ldg", "tma"])
@pytest.mark.parametrize("pro,epi,nb", INSTANCES)
def test_block_hot_exact(pro, epi, nb, impl, scales):
    """One hot block per token, in the first, a middle and the last (partial) segment over three launches, at 19 and 3 segments
    (the TMA kernel at 8 tokens: 3 only). STORE: bitwise with
    power-of-two scales, within three f32 roundings otherwise; RESIDUAL: x0 + that in f32; SWIGLU: act(gate) * up of those."""
    sms = _device_sms()
    for n in HOT_N:
        if (impl, n, nb) in TMA_REFUSES:
            assert plan_of(pro, epi, nb, HOT_D, n, sms, impl).rc == 1
            continue
        assert_plan(pro, epi, nb, HOT_D, n, sms, impl, 2 if impl == "tma" else 1)
        _block_hot(hot_matrix(n, scales), pro, epi, nb, impl, scales, sms)


def _block_hot(W, pro, epi, nb, impl, scales, sms):
    x0 = torch.randn(nb, W.d, device="cuda", generator=gen("hot-x0", nb))
    for rnd in range(3):
        x, nw, blocks, ks, hs = hot_inputs(nb, W.n, rnd, pro, scales == "pow2", 1)
        got = run_q40(W, x, pro, epi, nw=nw if pro == RMS else None, x0=x0, impl=impl, sms=sms, eps=0.0)
        ref, tol = hot_ref(W, blocks, ks, hs)
        what = f"block-hot {W.d}x{W.n} {impl} pro={pro} epi={epi} nb={nb} {scales} round {rnd} blocks {blocks}"
        exact = scales == "pow2"
        if epi == STORE:
            if exact:
                assert torch.equal(got.double(), ref), what
            else:
                assert_within(got, ref, tol, what)
        elif epi == RESID:
            if exact:
                assert torch.equal(got, x0 + ref.float()), what
            else:
                r = x0.double() + ref
                assert_within(got, r, tol + C_SUM * (x0.double().abs() + r.abs()), what)
        else:
            h, eh = glu_ref(ref, tol, SILU)
            assert_within(got, h, eh, what)


# ---- random data against float64 -----------------------------------------------------------------------------------------
SMALL = [(256, 256), (6144, 4096), (4096, 1792), (1000, 2176), (128, 768), (16032, 4096), (402, 14336), (512, 1024),
         (200, 4096),        # fewer pairs than SMs: one pair per CTA, half-empty 4-row groups on the TMA kernel
         (1000, 18560),      # 19 segments, the last one partial
         (1000, 4160)]       # n % 128 != 0: per-thread loads only
_CASES = {}


def matrix(d, n, seed=0):
    if (d, n, seed) not in _CASES:
        _CASES.clear()
        _CASES[d, n, seed] = Q40(d, n, seed)
    return _CASES[d, n, seed]


def _note(kernel, r):
    RATIOS[kernel] = max(RATIOS.get(kernel, 0.0), r)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["ldg", "tma"])
@pytest.mark.parametrize("d,n", SMALL)
def test_random_every_instance(d, n, impl):
    """Random weights and inputs on every instantiated (pro, epi, nb), SwiGLU with SiLU and GELU."""
    sms = _device_sms()
    W = matrix(d, n)
    x, nw, x0 = inputs(8, n, d, 0)
    for pro, epi, nb in INSTANCES:
        if (impl, n, nb) in TMA_REFUSES and d == HOT_D:
            assert plan_of(pro, epi, nb, d, n, sms, "tma").rc == 1 and plan_of(pro, epi, nb, d, n, sms).kernel == 1
            continue
        if impl == "tma" and n % 128:
            assert plan_of(pro, epi, nb, d, n, sms, "tma").rc == 1
            assert plan_of(pro, epi, nb, d, n, sms).kernel == 1
            with pytest.raises(RuntimeError, match="code 1"):
                run_q40(W, x[:nb], pro, epi, nw=nw, x0=x0, impl="tma", sms=sms)
            continue
        assert_plan(pro, epi, nb, d, n, sms, impl, 2 if impl == "tma" else 1)
        for act_fn in ((SILU, GELU) if epi == SWIGLU else (SILU,)):
            got = run_q40(W, x[:nb], pro, epi, nw=nw if pro == RMS else None, x0=x0, impl=impl, sms=sms, act_fn=act_fn)
            _note(impl, check_q40(W, x[:nb], pro, epi, got, nw=nw, x0=x0, act_fn=act_fn,
                                  what=f"{d}x{n} {impl} pro={pro} epi={epi} nb={nb} act={act_fn}"))


# (d, n, pro, epi, nb, impl, sms, kernel, stageRows, nStages, launches): ring wraps, one-stage rings and forced splits
GEOMETRY = [
    (6144, 4096, RMS, STORE, 1, "tma", 7, 2, 16, 2, 1),       # 878-row tiles through a 2-stage ring: 55 fills per CTA
    (6144, 4096, PLAIN, RESID, 8, "tma", 7, 2, 16, 2, 1),     # the same ring with 8 token planes
    (4096, 4096, RMS, SWIGLU, 8, "auto", 2, 2, 16, 2, 2),     # 2048-row tiles: no kernel holds 8 tokens, two TMA launches of 4
    (4096, 4096, PLAIN, RESID, 8, "ldg", 2, 1, 0, 0, 2),      # the same split on the per-thread-load kernel
    (4096, 4096, RMS, STORE, 8, "auto", 2, 2, 16, 2, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEOMETRY, ids=lambda c: f"{c[0]}x{c[1]}-epi{c[3]}-nb{c[4]}-{c[5]}-{c[6]}sms")
def test_ring_and_split_geometry(case):
    d, n, pro, epi, nb, impl, sms, kernel, sr, st, launches = case
    p = assert_plan(pro, epi, nb, d, n, sms, impl, kernel, launches)
    assert (p.stage_rows, p.n_stages) == (sr, st), p
    W = matrix(d, n, 1)
    x, nw, x0 = inputs(nb, n, d, 1)
    got = run_q40(W, x, pro, epi, nw=nw, x0=x0, impl=impl, sms=sms)
    _note({1: "ldg", 2: "tma"}[kernel], check_q40(W, x, pro, epi, got, nw=nw, x0=x0, what=f"geometry {case}"))


PRODUCTION = [("llama-3.1-8b", "logits"), ("qwen3-14b", "w2"), ("qwen3-14b", "logits"), ("llama-3.3-70b", "logits"),
              ("llama-3.3-70b", "w2"), ("llama-3.3-70b", "w13")]


@pytest.mark.gpu
@pytest.mark.parametrize("model,mat", PRODUCTION)
def test_production_shapes(model, mat):
    """The engine's epilogue at nb 1, 2, 4, 8 through impl "auto": Llama-3.1-8B logits (one-stage ring at nb 8), Qwen3-14B W2
    (nseg 17; TMA to nb 4, per-thread loads at 8), Llama-3.3-70B W1|W3 (same switch), and the three shapes whose 8-token
    batches run as two launches. On a 132-SM device each launch must take its pinned plan."""
    d, n = MODELS[model][mat]
    pro, epi = MATRIX[mat]
    sms = _device_sms()
    W = matrix(d, n, 2)
    x, nw, x0 = inputs(8, n, d, 2)
    for nb, want in zip(NBS, PLAN_TABLE.get(sms, PLAN_TABLE[132])[model][mat].split()):
        p = plan_of(pro, epi, nb, d, n, sms)
        if sms in PLAN_TABLE:
            assert _fmt(p) == want, (model, mat, nb, p)
        got = run_q40(W, x[:nb], pro, epi, nw=nw, x0=x0, sms=sms)
        _note({1: "ldg", 2: "tma"}[p.kernel], check_q40(W, x[:nb], pro, epi, got, nw=nw, x0=x0,
                                                        what=f"{model} {mat} nb={nb} plan {_fmt(p)}"))


# ---- layout and invariants -----------------------------------------------------------------------------------------------
def _nan_payload(shape):
    return torch.full(shape, NAN_F32, dtype=torch.int32, device="cuda").view(torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["ldg", "tma", "split"])
@pytest.mark.parametrize("epi", [STORE, RESID, SWIGLU])
def test_strides_repeat_and_token_independence(epi, impl):
    """inStride > n with NaN padding the kernel must not read; outStride > d with a NaN payload whose bits must survive; two
    launches bitwise equal; row t of an 8-token launch bitwise equal to a one-token launch of that row on the same kernel
    ("split": 8 tokens as two launches of 4, at 2 SMs)."""
    d, n = (4096, 4096) if impl == "split" else (1000, 2176)
    sms = 2 if impl == "split" else _device_sms()
    pro = PLAIN if epi == RESID else RMS
    kimpl = "auto" if impl == "split" else impl
    nb = 8
    assert_plan(pro, epi, nb, d, n, sms, kimpl, 1 if impl == "ldg" else 2, 2 if impl == "split" else 1)
    W = matrix(d, n, 3)
    x, nw, x0 = inputs(nb, n, d, 3)
    xin = torch.full((nb, n + 96), float("nan"), device="cuda")
    xin[:, :n] = x
    cols = out_cols(epi, d)
    base = _nan_payload((nb, cols + 40))

    def launch(rows):
        out = base[rows].clone()
        if epi == RESID:
            out[:, 8:8 + cols] = x0[rows]
        view = out[:, 8:8 + cols]
        _ops().gemv_q40(W.device(), xin[rows], pro=pro, epi=epi, out=view, norm_w=nw, eps=EPS, num_sms=sms, impl=kimpl)
        torch.cuda.synchronize()
        return out

    full = launch(slice(0, nb))
    bits = full.view(torch.int32)
    assert (bits[:, :8] == NAN_F32).all() and (bits[:, 8 + cols:] == NAN_F32).all(), "payload around the outputs overwritten"
    check_q40(W, x, pro, epi, full[:, 8:8 + cols], nw=nw, x0=x0, what=f"strided {impl} epi={epi}")
    assert torch.equal(bits, launch(slice(0, nb)).view(torch.int32)), "two launches differ"
    for t in range(nb):
        if impl == "split":
            break               # the one-token plan at 2 SMs is another kernel geometry
        one = launch(slice(t, t + 1))
        assert torch.equal(one.view(torch.int32), bits[t:t + 1]), f"token {t}: 8-token launch differs from a one-token launch"


# ---- arg-max ------------------------------------------------------------------------------------------------------------
AD, AN = 5000, 2048


class ArgBufs:
    def __init__(self, sms, cap):
        z = dict(device="cuda")
        self.val = torch.full((sms,), float("nan"), **z)
        self.idx = torch.full((sms,), -1, dtype=torch.int32, **z)
        self.counter = torch.zeros(4, dtype=torch.int32, **z)
        self.counter[1:] = 0x7eadbeef
        self.token = torch.full((1,), -1, dtype=torch.int32, **z)
        self.pos = torch.zeros(1, dtype=torch.int32, **z)
        self.history = torch.full((cap + 8,), -7, dtype=torch.int32, **z)


def argmax_call(W, x, nw, bufs, *, cap, row_offset=0, vocab_limit=0, sms):
    out = torch.full((W.d,), float("nan"), device="cuda")
    _ops().gemv_q40_argmax(W.device(), x, norm_w=nw, eps=EPS, out=out, arg_val=bufs.val, arg_idx=bufs.idx, arg_counter=bufs.counter,
                           token=bufs.token, pos=bufs.pos, history=bufs.history, history_cap=cap, row_offset=row_offset,
                           vocab_limit=vocab_limit, num_sms=sms)
    torch.cuda.synchronize()
    return out


def lowest_max(v):
    m = v.max()
    return int((v == m).nonzero()[0])


@pytest.mark.gpu
@pytest.mark.parametrize("row_offset,limit_at", [(0, None), (0, 4321), (96000, 1200)])
def test_fused_argmax(row_offset, limit_at):
    """Logits bitwise those of the RMSNORM/STORE one-token TMA launch; the token is the lowest-index maximum of those logits among
    global ids < vocabLimit, with a maximum tied bitwise over rows of different CTAs and (limit_at) a larger one planted at or
    above the limit; pos advances and history[pos] is written only below historyCap; a second launch is right too."""
    sms = _device_sms()
    W = Q40(AD, AN, 7)
    x, nw, _ = inputs(1, AN, AD, 7)
    x = x[0]
    probe = run_q40(W, x[None], RMS, STORE, nw=nw, impl="tma", sms=sms)[0]
    m = lowest_max(probe)
    blk = AN // 32
    tied = sorted({17, AD // 3, m, AD - 2})                 # 17 and AD / 3 lie in other CTAs than m at any SM count here
    for r in tied:
        W.raw[r * blk:(r + 1) * blk] = W.raw[m * blk:(m + 1) * blk]
    if limit_at is not None:
        hi = limit_at + 5
        sc = W.raw[m * blk:(m + 1) * blk, :2].clone().view(torch.float16) * 2
        W.raw[hi * blk:(hi + 1) * blk] = W.raw[m * blk:(m + 1) * blk]
        W.raw[hi * blk:(hi + 1) * blk, :2] = sc.view(torch.uint8)
    W._dev = None
    assert plan_of(RMS, 3, 1, AD, AN, sms, "tma").rc == 0
    store = run_q40(W, x[None], RMS, STORE, nw=nw, impl="tma", sms=sms)[0]
    assert (store[tied] == store[tied[0]]).all() and probe[m] > 0
    limit = 0 if limit_at is None else row_offset + limit_at
    if limit_at is not None:
        assert store[limit_at + 5] > store[tied[0]], "planted maximum above the limit is not the largest logit"
    local_lim = AD if limit_at is None else limit_at
    want = row_offset + lowest_max(store[:local_lim])
    assert want == row_offset + tied[0]
    for cap, p0 in ((40, 10), (11, 10)):
        bufs = ArgBufs(sms, 64)
        bufs.pos[0] = p0
        for call in range(2):
            logits = argmax_call(W, x, nw, bufs, cap=cap, row_offset=row_offset, vocab_limit=limit, sms=sms)
            what = f"argmax offset={row_offset} limit={limit} cap={cap} call {call}"
            assert torch.equal(logits.view(torch.int32), store.view(torch.int32)), f"{what}: logits differ from the STORE launch"
            assert int(bufs.token[0]) == want, f"{what}: token {int(bufs.token[0])}, expected {want}"
            p = p0 + 1 + call
            assert int(bufs.pos[0]) == p, what
            h = bufs.history.cpu()
            assert h[p] == (want if p < cap else -7), f"{what}: history[{p}] = {int(h[p])}"
            assert int(bufs.counter[0]) == 0 and (bufs.counter[1:] == 0x7eadbeef).all(), f"{what}: counter not reset"
        h = bufs.history.cpu()
        written = [i for i in range(len(h)) if h[i] != -7]
        assert written == [i for i in (p0 + 1, p0 + 2) if i < cap], (cap, written)


def _adv(logits, vocab, p0=3, cap=100):
    token = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    pos = torch.full((1,), p0, dtype=torch.int32, device="cuda")
    hist = torch.full((cap + 8,), -7, dtype=torch.int32, device="cuda")
    _ops().argmax_advance(logits, vocab, token, pos, hist, cap)
    torch.cuda.synchronize()
    return int(token[0]), int(pos[0]), hist.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("vocab", [1, 1023, 1024, 1025, 151936])
def test_argmax_advance(vocab):
    """Lowest index among the maxima with ties inside a thread, across threads of a warp and across warps; -inf entries; entries
    past vocab are ignored; pos advances and history[pos] is written below historyCap only."""
    g = gen("adv", vocab)
    buf = torch.full((vocab + 64,), 1e30, device="cuda")      # past the vocabulary: never read
    lg = torch.randn(vocab, device="cuda", generator=g)
    lg[torch.rand(vocab, device="cuda", generator=g) < 0.1] = float("-inf")
    ties = sorted({i for i in (vocab - 1, vocab // 2, 1029, 40, 6, 5) if i < vocab})
    lg[ties] = 9.0
    buf[:vocab] = lg
    tok, pos, h = _adv(buf, vocab)
    assert tok == ties[0] and pos == 4 and h[4] == ties[0] and (h[:4] == -7).all() and (h[5:] == -7).all()
    # no history past the cap
    tok, pos, h = _adv(buf, vocab, p0=9, cap=10)
    assert tok == ties[0] and pos == 10 and (h == -7).all()
    # every entry -inf but one finite in the last thread's range; then all -inf: index 0
    buf[:vocab] = float("-inf")
    buf[vocab - 1] = -3.0
    assert _adv(buf, vocab)[0] == vocab - 1
    buf[vocab - 1] = float("-inf")
    assert _adv(buf, vocab)[0] == 0


# ---- dense GEMV ---------------------------------------------------------------------------------------------------------
DENSE_COMBOS = [(p, e, nb) for (p, e), nbs in COMBOS.items() if (p, e) != (PLAIN, SWIGLU) for nb in nbs]


@pytest.mark.gpu
@pytest.mark.parametrize("wdt", ["f32", "f16"])
@pytest.mark.parametrize("d,n", [(640, 1032), (640, 1024), (6, 2056), (1000, 4104)])
def test_dense(d, n, wdt):
    """f32 and f16 weights on every (pro, epi, nb), SiLU and GELU, with input and output strides; n not a multiple of the unrolled
    chunk stride (1024 f32 / 2048 f16 values) and a d smaller than the SM count."""
    ops = _ops()
    dt = torch.float32 if wdt == "f32" else torch.float16
    g = gen("dense", d, n, wdt)
    w = (torch.randn(d, n, device="cuda", generator=g) / n ** 0.5).to(dt)
    Wd = ops.DeviceDense(w, d, n)
    w64 = w.double()
    xin = torch.full((8, n + 24), float("nan"), device="cuda")
    xin[:, :n] = torch.randn(8, n, device="cuda", generator=g)
    x = xin[:, :n]
    nw = torch.rand(n, device="cuda", generator=g) + 0.5
    x0 = torch.randn(8, d, device="cuda", generator=g)
    chain = (n / 32 + 6) * 2.0 ** -24
    for pro, epi, nb in DENSE_COMBOS:
        y = rms64(x[:nb], nw, EPS) if pro == RMS else x[:nb].double()
        ref = y @ w64.T
        tol = ((REL_NORM if pro == RMS else 0.0) + chain) * (y.abs() @ w64.abs().T)
        for act_fn in ((SILU, GELU) if epi == SWIGLU else (SILU,)):
            cols = out_cols(epi, d)
            out = _nan_payload((nb, cols + 16))
            if epi == RESID:
                out[:, :cols] = x0[:nb]
            ops.gemv_dense(Wd, x[:nb], pro=pro, epi=epi, out=out[:, :cols], norm_w=nw, eps=EPS, act_fn=act_fn)
            torch.cuda.synchronize()
            assert (out.view(torch.int32)[:, cols:] == NAN_F32).all(), "payload past the outputs overwritten"
            what = f"dense {wdt} {d}x{n} pro={pro} epi={epi} nb={nb} act={act_fn}"
            got = out[:, :cols]
            if epi == STORE:
                r = assert_within(got, ref, tol, what)
            elif epi == RESID:
                rr = x0[:nb].double() + ref
                r = assert_within(got, rr, tol + C_SUM * (x0[:nb].double().abs() + rr.abs()), what)
            else:
                r = assert_within(got, *glu_ref(ref, tol, act_fn), what)
            _note("dense", r)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nlargest error / bound per kernel:", {k: round(v, 4) for k, v in sorted(RATIOS.items())})
