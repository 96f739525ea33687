"""The q80 KV cache (`--kv-cache-float-type q80`): int8 value planes with one f16 scale per 32 values in a separate plane.

* Writer: ropeKvKernel's stored ints and scales against q80 of a float64 QK-norm + RoPE of the same row. The kernel rounds in
  f32, so where x / d lies within a hair of a rounding boundary either neighbour is accepted (the bracket of test_gpu_moe.py).
* Every decode-attention kernel over q80 caches against float64 attention over the dequantised cache, bound 2e-4 * max|V|, with
  the needle keys of test_gpu_slots.py at split boundaries and in the neighbouring slots.
* Prefill attention over q80 caches, on the tensor cores and on the per-token fallback: test_gpu_attn_prefill.py, where the cache
  type is a parameter of every case (the reference widens the tiles to bf16 as the kernel does).
* The engine on q80 against OracleModel(kv_quant="q80") for every tiny family; the slots and choices steps; the persistent kernel
  against the multi-kernel path at Llama-3.1-8B layer shapes; slots batch invariance; both command-line stacks.
"""
import dataclasses
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_V = 2e-4
N_SPLITS = 8
NEEDLE_SCORE = 30.0


def q80_quant(x: torch.Tensor):
    """x [..., hd] (f32) -> (int8 values, f16 scales [..., hd / 32]) with the kernels' f32 arithmetic."""
    g = x.float().reshape(*x.shape[:-1], -1, 32)
    d = g.abs().amax(dim=-1, keepdim=True) / 127.0
    inv = torch.where(d != 0, 1.0 / d, torch.zeros_like(d))
    q = torch.round(g * inv).to(torch.int8)   # half-to-even like __float2int_rn
    return q.reshape(x.shape), d.squeeze(-1).half()


def q80_dequant(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    g = q.double().reshape(*q.shape[:-1], -1, 32) * s.double().unsqueeze(-1)
    return g.reshape(q.shape)


def _planes(x: torch.Tensor):
    """Device int8 values and padded f16 scale plane of the cache x [nKv, L, hd]."""
    q, s = q80_quant(x)
    sp = torch.zeros(s.numel() + 8, dtype=torch.float16)
    sp[:s.numel()] = s.reshape(-1)
    return q.cuda().contiguous(), sp.cuda(), q80_dequant(q, s)


def _split_bounds(p: int):
    n_pos = p + 1
    eff = max(1, min(N_SPLITS, (n_pos + 63) // 64))
    chunk = (n_pos + eff - 1) // eff
    return [s * chunk for s in range(1, eff) if s * chunk < n_pos]


def _attn_ref(q, K, V, n, scale):
    s = (K[:n] @ q.double()) * scale
    return torch.softmax(s, dim=0) @ V[:n]


# ---- writer ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hd", [64, 128])
def test_rope_kv_writer_matches_q80_ref(hd):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    g = torch.Generator().manual_seed(hd)
    n_heads, n_kv, L, nb, eps = 8, 2, 96, 6, 1e-6
    qkv_dim = (n_heads + 2 * n_kv) * hd
    qkv = torch.randn(nb, qkv_dim, generator=g) * 3
    qkv[0, n_heads * hd:(n_heads + 1) * hd] = 0.0                # an all-zero K row: scale 0, values 0
    pos = [0, 5, 31, 64, 90, 95]
    ang = torch.rand(L, hd // 2, generator=g, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1).float()
    q_norm = torch.rand(hd, generator=g) + 0.5
    k_norm = torch.rand(hd, generator=g) + 0.5
    kq = torch.zeros(n_kv, L, hd, dtype=torch.int8, device="cuda")
    vq = torch.zeros_like(kq)
    ks = torch.zeros(n_kv * L * hd // 32 + 8, dtype=torch.float16, device="cuda")
    vs = torch.zeros_like(ks)
    qd = qkv.cuda().contiguous()
    posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
    rd, qn, kn = rope.cuda().contiguous(), q_norm.cuda(), k_norm.cuda()
    assert lib.dl_rope_kv_q80(qd.data_ptr(), qkv_dim, posd.data_ptr(), rd.data_ptr(), qn.data_ptr(), kn.data_ptr(), eps, n_heads, n_kv, hd, L,
                              kq.data_ptr(), vq.data_ptr(), ks.data_ptr(), vs.data_ptr(), nb, cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    kq, vq = kq.cpu(), vq.cpu()
    ks = ks[:n_kv * L * hd // 32].cpu().reshape(n_kv, L, hd // 32)
    vs = vs[:n_kv * L * hd // 32].cpu().reshape(n_kv, L, hd // 32)
    worst = 0.0
    for t, p in enumerate(pos):
        row = qkv[t].double()
        cs = rope[p].double()
        for h in range(n_kv):
            k = row[(n_heads + h) * hd:(n_heads + h + 1) * hd]
            k = k_norm.double() * (k / torch.sqrt((k * k).mean() + eps))
            a, b = k[0::2].clone(), k[1::2].clone()
            k[0::2], k[1::2] = a * cs[:, 0] - b * cs[:, 1], a * cs[:, 1] + b * cs[:, 0]
            v = row[(n_heads + n_kv + h) * hd:(n_heads + n_kv + h + 1) * hd]
            for x, qs, ss in ((k, kq[h, p], ks[h, p]), (v, vq[h, p], vs[h, p])):
                xb = x.reshape(-1, 32)
                d = xb.abs().amax(dim=1) / 127.0
                # the scale: f16 of the f32 amax / 127 (one f16 step of slack for the f32 rounding of the inputs)
                want_s = d.half().double()
                got_s = ss.double()
                assert torch.all((got_s - want_s).abs() <= want_s * 2 ** -10 + 1e-30), (t, h, got_s, want_s)
                # the ints: rint(x / d), either neighbour where x / d is within a hair of a .5 boundary
                ratio = torch.where(d[:, None] > 0, xb / d[:, None].clamp_min(1e-300), torch.zeros_like(xb)).reshape(-1)
                dev_ = (qs.double() - ratio).abs()
                worst = max(worst, dev_.max().item())
                assert torch.all(dev_ <= 0.5 + 1e-3), (t, h, dev_.max().item())
                assert torch.all(qs.abs() <= 127)
    assert int(kq[0, 0].abs().sum()) == 0 and float(ks[0, 0].abs().sum()) == 0.0   # the zero row
    assert worst > 0.4                                                              # the ints are rounded, not truncated


# ---- decode attention ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4), (64, 4), (128, 1)])
@pytest.mark.parametrize("nb", [1, 3, 8])
def test_attn_decode_q80_matches_float64(nb, hd, kv_mul):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    g = torch.Generator().manual_seed(nb * 7 + hd + kv_mul)
    n_kv, L = 2, 1100
    n_heads = n_kv * kv_mul
    q_dim = n_heads * hd
    qkv_dim = q_dim + 2 * n_kv * hd
    pos = [[0, 63, 64, 513, 1099, 300, 127, 700][(b * 5 + hd // 64) % 8] for b in range(nb)]
    qkv = torch.randn(nb, qkv_dim, generator=g)
    k = torch.randn(n_kv, L, hd, generator=g) * 0.6
    v = torch.randn(n_kv, L, hd, generator=g)
    kq, ks, K = _planes(k)
    vq, vs, V = _planes(v)
    qd = qkv.cuda().contiguous()
    posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
    partial = torch.zeros(nb * n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(nb * n_heads, dtype=torch.int32, device="cuda")
    out = torch.full((nb, q_dim), float("nan"), device="cuda")
    assert lib.dl_attn_decode_q80(qd.data_ptr(), qkv_dim, posd.data_ptr(), kq.data_ptr(), vq.data_ptr(), ks.data_ptr(), vs.data_ptr(), n_heads,
                                  n_kv, hd, L, N_SPLITS, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim, None, nb, cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    got = out.cpu().double()
    scale = 1.0 / math.sqrt(hd)
    for b in range(nb):
        for h in range(n_heads):
            kvh = h // kv_mul
            want = _attn_ref(qkv[b, h * hd:(h + 1) * hd], K[kvh], V[kvh], pos[b] + 1, scale)
            err = (got[b, h * hd:(h + 1) * hd] - want).abs().max().item()
            bound = TOL_V * V[kvh, :pos[b] + 1].abs().max().item()
            assert err <= bound, (b, h, pos[b], err, bound)


@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4)])
@pytest.mark.parametrize("p", [0, 40, 64, 700, 1023])
def test_attn_fused_q80_matches_float64(p, hd, kv_mul):
    """The fused single-token kernel appends the token's row in q80 and attends to it as stored."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    g = torch.Generator().manual_seed(p + hd)
    n_kv, L = 2, 1024
    n_heads = n_kv * kv_mul
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    qkv = torch.randn(q_dim + 2 * kv_dim, generator=g)
    rope = torch.zeros(L, hd // 2, 2)
    rope[..., 0] = 1.0                                             # identity rotation: the reference needs no RoPE
    k = torch.randn(n_kv, L, hd, generator=g) * 0.6
    v = torch.randn(n_kv, L, hd, generator=g)
    kq, ks, _ = _planes(k)
    vq, vs, _ = _planes(v)
    qd = qkv.cuda()
    posd = torch.tensor([p], dtype=torch.int32, device="cuda")
    partial = torch.zeros(n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(n_heads, dtype=torch.int32, device="cuda")
    out = torch.full((q_dim,), float("nan"), device="cuda")
    rd = rope.cuda().contiguous()
    assert lib.dl_attn_fused_q80(qd.data_ptr(), posd.data_ptr(), rd.data_ptr(), None, None, 1e-6, kq.data_ptr(), vq.data_ptr(), ks.data_ptr(),
                                 vs.data_ptr(), n_heads, n_kv, hd, L, N_SPLITS, partial.data_ptr(), counters.data_ptr(), out.data_ptr(),
                                 cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    n_sc = n_kv * L * hd // 32
    K = q80_dequant(kq.cpu(), ks[:n_sc].cpu().reshape(n_kv, L, hd // 32))
    V = q80_dequant(vq.cpu(), vs[:n_sc].cpu().reshape(n_kv, L, hd // 32))
    for h in range(n_kv):                                          # the new row is q80 of the raw k / v
        for X, src in ((K, qkv[q_dim + h * hd:q_dim + (h + 1) * hd]), (V, qkv[q_dim + kv_dim + h * hd:q_dim + kv_dim + (h + 1) * hd])):
            want = q80_dequant(*q80_quant(src[None]))[0]
            assert (X[h, p] - want).abs().max().item() <= 1.01 * want.abs().max().item() / 127 / 2 + 1e-6
    got = out.cpu().double()
    scale = 1.0 / math.sqrt(hd)
    for h in range(n_heads):
        kvh = h // kv_mul
        want = _attn_ref(qkv[h * hd:(h + 1) * hd], K[kvh], V[kvh], p + 1, scale)
        err = (got[h * hd:(h + 1) * hd] - want).abs().max().item()
        assert err <= TOL_V * V[kvh, :p + 1].abs().max().item(), (h, err)


@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4), (64, 4), (128, 1)])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_slot_attention_q80_matches_float64(B, hd, kv_mul):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    L = 1024
    g = torch.Generator().manual_seed(B * 17 + hd + kv_mul * 3)
    n_kv = 2
    n_heads = n_kv * kv_mul
    q_dim = n_heads * hd
    qkv_dim = q_dim + 2 * n_kv * hd
    choices = [0, 63, 64, 300, L - 1, 511, 127, 700]
    pos = [choices[(b * 3 + hd // 64) % len(choices)] for b in range(B)]
    inactive = 0b10 if B >= 3 else 0
    qkv = torch.randn(B, qkv_dim, generator=g)
    k = torch.randn(B, n_kv, L, hd, generator=g) * 0.6
    v = torch.randn(B, n_kv, L, hd, generator=g)
    scale = 1.0 / math.sqrt(hd)
    for b in range(B):
        q0 = qkv[b, :hd].double()
        needle = (q0 * (NEEDLE_SCORE / (scale * float(q0 @ q0)))).float()
        for r in [0, pos[b]] + _split_bounds(pos[b]) + [x - 1 for x in _split_bounds(pos[b])]:
            k[b, 0, r] = needle * 0.5
        for nb_ in (b - 1, b + 1):
            if 0 <= nb_ < B:
                for r in {0, pos[b] // 2, pos[b]}:
                    k[nb_, 0, r] = needle
    kq, ks, K = _planes(k)                                         # slot b at element offset b * n_kv * L * hd of both planes
    vq, vs, V = _planes(v)
    qd = qkv.cuda().contiguous()
    posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
    partial = torch.zeros(B * n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(B * n_kv, dtype=torch.int32, device="cuda")
    out = torch.full((B, q_dim), float("nan"), device="cuda")
    assert lib.dl_slot_attn_q80(qd.data_ptr(), qkv_dim, posd.data_ptr(), kq.data_ptr(), vq.data_ptr(), ks.data_ptr(), vs.data_ptr(), n_heads,
                                n_kv, hd, L, N_SPLITS, B, inactive, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim,
                                cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    got = out.cpu().double()
    assert int(counters.abs().sum()) == 0
    for b in range(B):
        if (inactive >> b) & 1:
            continue
        for h in range(n_heads):
            kvh = h // kv_mul
            want = _attn_ref(qkv[b, h * hd:(h + 1) * hd], K[b, kvh], V[b, kvh], pos[b] + 1, scale)
            err = (got[b, h * hd:(h + 1) * hd] - want).abs().max().item()
            bound = TOL_V * V[b, kvh, :pos[b] + 1].abs().max().item()
            assert err <= bound, (b, h, pos[b], err, bound)


@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4)])
@pytest.mark.parametrize("B,P,j", [(1, 0, 0), (4, 130, 3), (8, 600, 7), (3, 64, 1)])
def test_choice_attention_q80_matches_float64(B, P, j, hd, kv_mul):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    g = torch.Generator().manual_seed(B + P + hd)
    n_kv, C = 2, 8
    L = P + 1 + B * C + 5
    n_heads = n_kv * kv_mul
    q_dim = n_heads * hd
    qkv_dim = q_dim + 2 * n_kv * hd
    mask = 0b10 if B >= 3 else 0
    qkv = torch.randn(B, qkv_dim, generator=g)
    k = torch.randn(n_kv, L, hd, generator=g) * 0.6
    v = torch.randn(n_kv, L, hd, generator=g)
    scale = 1.0 / math.sqrt(hd)
    if B > 1:                                                      # choice 1's own row: choice 0 must not see it
        q0 = qkv[0, :hd].double()
        k[0, P + 1 + C] = (q0 * (NEEDLE_SCORE / (scale * float(q0 @ q0)))).float()
    kq, ks, K = _planes(k)
    vq, vs, V = _planes(v)
    qd = qkv.cuda().contiguous()
    partial = torch.zeros(B * n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(n_kv, dtype=torch.int32, device="cuda")
    out = torch.full((B, q_dim), float("nan"), device="cuda")
    assert lib.dl_choice_attn_only_q80(qd.data_ptr(), qkv_dim, kq.data_ptr(), vq.data_ptr(), ks.data_ptr(), vs.data_ptr(), n_heads, n_kv, hd, L,
                                       N_SPLITS, B, P, C, j, mask, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim,
                                       cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    got = out.cpu().double()
    for b in range(B):
        if (mask >> b) & 1:
            continue
        rows = list(range(P + 1)) + list(range(P + 1 + b * C, P + 1 + b * C + j + 1))
        for h in range(n_heads):
            kvh = h // kv_mul
            Kb, Vb = K[kvh, rows], V[kvh, rows]
            want = _attn_ref(qkv[b, h * hd:(h + 1) * hd], Kb, Vb, len(rows), scale)
            err = (got[b, h * hd:(h + 1) * hd] - want).abs().max().item()
            bound = TOL_V * Vb.abs().max().item()
            assert err <= bound, (b, h, err, bound)


# ---- engine ----------------------------------------------------------------------------------------------------------------------

def _engine(path, **kw):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    return Engine(load_device_weights(ModelFile(path)), kv_cache_float_type="q80", **kw)


def _oracle(path):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.reference import OracleModel
    return OracleModel(ModelFile(path), act_quant="q80", device="cuda", kv_quant="q80")


def test_unknown_kv_cache_type_is_refused(tmp_models):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    with pytest.raises(ValueError, match="KV-cache float type"):
        Engine(load_device_weights(ModelFile(tmp_models["tiny-llama"][0])), kv_cache_float_type="fp8")


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-llama31", "tiny-qwen3", "tiny-qwen3-moe"])
def test_engine_q80_matches_oracle(tmp_models, name):
    """Token by token, and a batched prefill then decode, on q80 caches against the oracle that rounds its stored K/V rows the same
    way: test_engine_matches_oracle's sequence, paths and tolerance (the tensor-core prefill has its float64 test in test_gpu_attn_prefill.py)."""
    path = tmp_models[name][0]
    toks = [3, 17, 250, 9, 44, 101, 7, 300, 12, 5, 77]
    ref = _oracle(path).forward(toks, 0)
    eng = _engine(path)
    for i, t in enumerate(toks):
        err = (eng.step(t, i) - ref[i]).abs().max().item()
        assert err < 0.06, f"pos {i}: {err}"
    eng2 = _engine(path)
    eng2.use_tc_prefill = False
    P = 8
    lg = eng2.prefill(toks[:P], 0)
    assert (lg - ref[P - 1]).abs().max().item() < 0.06
    for i in range(P, len(toks)):
        assert (eng2.step(toks[i], i) - ref[i]).abs().max().item() < 0.06, i


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-llama31", "tiny-qwen3"])
def test_slots_step_q80_matches_oracle(tmp_models, name):
    """Teacher-forced rows against the q80 oracle with test_gpu_slots.py's rule: within test_engine_matches_oracle's tolerance, or,
    where the single-sequence q80 engine (same prefill kernels, then one token per step) is itself further from the oracle, within
    that engine's error plus a margin; and close to that engine. "Close" is 3e-2 rather than the bf16 test's 1e-2: the two paths
    round K/V rows whose f32 values differ in the last bits, and a one-step q80 flip is 1/127 of the block's largest value."""
    path = tmp_models[name][0]
    N = 4
    eng = _engine(path)
    eng.set_slots(N)
    prompts = [[(11 * b + 7 * i + 3) % 500 + 1 for i in range(4 + 5 * b)] for b in range(N)]
    follow = [[(5 * b + 13 * j) % 400 + 2 for j in range(5)] for b in range(N)]
    ref, single = [], []
    for b in range(N):
        seq = prompts[b] + follow[b]
        P = len(prompts[b]) - 1
        ref.append(_oracle(path).forward(seq, 0)[P:])
        one = _engine(path)
        one.tc_min_tokens = 1
        one.prefill(seq[:P], 0, want_logits=False)
        single.append([one.step(seq[p], p).clone() for p in range(P, len(seq))])
        eng.slot_prefill(b, prompts[b][:-1], 0)
    tokens = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    for j in range(len(follow[0]) + 1):
        lg = eng.slots_forward(tokens, pos, [True] * N).clone()
        for b in range(N):
            err = (lg[b] - ref[b][j]).abs().max().item()
            base = (single[b][j] - ref[b][j]).abs().max().item()
            assert err < max(0.06, base + 0.03), (b, j, err, base)
            assert (lg[b] - single[b][j]).abs().max().item() < 3e-2, (b, j)
            if j < len(follow[b]):
                tokens[b], pos[b] = follow[b][j], pos[b] + 1
    # slot_copy moves both planes: a copy of slot 0's prompt continues exactly like slot 0
    eng.slot_copy(0, 3, len(prompts[0]) - 1)
    t = [prompts[0][-1]] * 4
    p = [len(prompts[0]) - 1] * 4
    eng.slot_copy(0, 1, len(prompts[0]) - 1)
    lg = eng.slots_forward(t, p, [False, True, False, True]).clone()
    assert torch.equal(lg[1], lg[3])
    assert (lg[1] - single[0][0]).abs().max().item() < 3e-2


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-llama31", "tiny-qwen3"])
def test_choices_step_q80_matches_oracle(tmp_models, name):
    path = tmp_models[name][0]
    eng = _engine(path)
    prompt = [3, 17, 250, 9, 44, 101, 7, 300, 12, 5]
    P = len(prompt) - 1
    n, C = 3, 6
    forced = [[(7 * b + 3 * j) % 400 + 5 for j in range(4)] for b in range(n)]
    eng.tc_min_tokens = 1
    eng.prefill(prompt[:P], 0, want_logits=False)
    eng.step(prompt[P], P)
    refs = [_oracle(path).forward(prompt + forced[b], 0) for b in range(n)]
    assert (eng.logits[0] - refs[0][P]).abs().max().item() < 0.06
    for j in range(len(forced[0])):
        eng.choices_forward([forced[b][j] for b in range(n)], P, C, j)
        lg = eng.logits[:n].clone()
        for b in range(n):
            err = (lg[b] - refs[b][P + 1 + j]).abs().max().item()
            assert err < 0.06, (b, j, err)


def test_slots_q80_batch_invariance(tmp_models):
    """On q80 caches too, a row's logits and draws are bit for bit those of the same sequence stepped alone."""
    N = 8
    eng = _engine(tmp_models["tiny-llama31"][0])
    eng.set_slots(N)
    prompts = [[(11 * b + 7 * i + 3) % 500 + 1 for i in range(4 + 5 * b)] for b in range(N)]
    steps = 10

    def run(rows):
        logits, drawn = {b: [] for b in rows}, {b: [] for b in rows}
        for b in rows:
            eng.slot_prefill(b, prompts[b][:-1], 0)
            eng.slot_sampling(b, 1000 + b, 0.8 if b % 2 else 0.0, 0.9)
        tokens = [prompts[b][-1] if b in rows else 0 for b in range(N)]
        pos = [len(prompts[b]) - 1 if b in rows else 0 for b in range(N)]
        active = [b in rows for b in range(N)]
        for _ in range(steps):
            out = eng.slots_step(tokens, pos, active)
            for b in rows:
                logits[b].append(eng.logits[b].cpu().clone())
                drawn[b].append(out[b])
                tokens[b], pos[b] = out[b], pos[b] + 1
        return logits, drawn

    all_lg, all_tok = run(list(range(N)))
    for b in (0, 5):
        lg, tok = run([b])
        assert tok[b] == all_tok[b], b
        for j in range(steps):
            assert torch.equal(lg[b][j], all_lg[b][j]), (b, j)


@pytest.fixture(scope="module")
def llama8b_layers(tmp_path_factory):
    """Llama-3.1-8B layer shapes (dim 4096, 32 q-heads, 8 KV heads of 128, ff 14336), 2 layers, small vocabulary."""
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    cfg = dataclasses.replace(get_config("llama-3.1-8b"), n_layers=2, max_seq_len=4096, vocab_size=4096)
    path = str(tmp_path_factory.mktemp("l8b") / "l8b.m")
    write_synthetic_model(path, cfg, seed=5)
    return path


def _mega_scale_skips(n_pos, n_splits, n_heads, n_kv, seq_len, hd):
    """Leading bytes the persistent kernel skips in the 16-byte aligned scale span of every K/V fill of one step (mega_decode.cu:
    attnSplits, AttnItem, kvScSkip); the scale plane itself starts 256-byte aligned."""
    eff = max(1, min(n_splits, (n_pos + 255) // 256))
    chunk = (n_pos + eff - 1) // eff
    skips = []
    for h in range(n_heads):
        kvh = h // (n_heads // n_kv)
        for split in range(eff):
            begin, end = split * chunk, min(split * chunk + chunk, n_pos)
            cached_end = end - 1 if end == n_pos else end
            for c0 in range(begin, cached_end, 64):
                skips.append(((kvh * seq_len * hd + c0 * hd) // 32 * 2) % 16)
    return skips


def test_persistent_kernel_q80_matches_multi_kernel(llama8b_layers):
    """With q80 caches the persistent kernel runs at Llama-3.1-8B shapes and agrees with the multi-kernel path step by step, from
    position 505 to 780. That crosses the split counts 2 -> 3 (nPos 513) and 3 -> 4 (nPos 769), where the splits start at odd rows,
    and the context of 4093 rows puts odd KV heads' scale planes 8 bytes off a 16-byte boundary: the fills copy aligned scale spans
    with 8 leading bytes to skip (asserted below from the kernel's rule). Afterwards all four cache planes written by the two paths
    are compared."""
    seq = 4093
    mega = _engine(llama8b_layers, seq_len=seq)
    multi = _engine(llama8b_layers, seq_len=seq)
    multi.enable_mega(False)
    w = mega.w
    p0, p1 = 505, 781
    toks = [(37 * i + 11) % 4000 + 1 for i in range(p1 + 1)]
    skips = [k for n in range(p0 + 1, p1 + 1) for k in _mega_scale_skips(n, mega.n_splits, w.n_heads, w.n_kv_heads, seq, w.header.head_dim)]
    assert 0 in skips and 8 in skips, sorted(set(skips))          # both the aligned and the offset scale spans are exercised
    for e in (mega, multi):
        e.prefill(toks[:p0], 0, want_logits=False)
    for p in range(p0, p1):
        a = mega.step(toks[p], p).clone()
        assert mega.mega_active, "the persistent kernel fell back to the multi-kernel path"
        b = multi.step(toks[p], p).clone()
        assert not multi.mega_active
        err = (a - b).abs().max().item()
        assert err < 2e-2 * b.abs().max().item() + 1e-3, (p, err)
    hd = w.header.head_dim
    n_sc = w.n_kv_heads * seq * hd // 32
    for l in range(w.header.n_layers):
        for name, vals, scales in (("K", "k_cache", "k_scale"), ("V", "v_cache", "v_scale")):
            vm, vn = getattr(mega, vals)[l], getattr(multi, vals)[l]
            sm = getattr(mega, scales)[l][:n_sc].view(w.n_kv_heads, seq, hd // 32).float()
            sn = getattr(multi, scales)[l][:n_sc].view(w.n_kv_heads, seq, hd // 32).float()
            # the prompt rows: the same prefill kernels on both engines
            assert torch.equal(vm[:, :p0], vn[:, :p0]) and torch.equal(sm[:, :p0], sn[:, :p0]), (l, name)
            # the decoded rows: written by megaAttention and by attnFusedKernel from q|k|v vectors of two different GEMVs (and, past
            # layer 0, of residual streams that already differ in the last bits), so a value may round one q80 step apart and a
            # scale a few f16 steps apart; the dequantised rows agree within a step. A scale written to the wrong row or block, or
            # read through a wrong span offset, is off by far more.
            dv = (vm[:, p0:p1].int() - vn[:, p0:p1].int()).abs()
            ds = (sm[:, p0:p1] - sn[:, p0:p1]).abs()
            assert dv.max().item() <= 1 and (dv == 0).float().mean().item() > 0.99, (l, name, dv.max().item())
            assert torch.all(ds <= sn[:, p0:p1].abs() * (2 ** -10 if l == 0 else 2 ** -7)), (l, name, ds.max().item())
            assert (sn[:, p0:p1] > 0).all(), (l, name)            # every decoded row got its scales
            deq_m = vm[:, p0:p1].float().view(w.n_kv_heads, p1 - p0, hd // 32, 32) * sm[:, p0:p1, :, None]
            deq_n = vn[:, p0:p1].float().view(w.n_kv_heads, p1 - p0, hd // 32, 32) * sn[:, p0:p1, :, None]
            # one q80 step of the row, plus |q| <= 127 times the scales' difference
            assert torch.all((deq_m - deq_n).abs() <= 1.01 * sn[:, p0:p1, :, None] + 127 * ds[..., None]), (l, name)
            # rows past the last decoded position are untouched
            assert int(vm[:, p1:].abs().sum()) == 0 and float(sm[:, p1:].abs().sum()) == 0.0, (l, name)


# ---- front-ends ------------------------------------------------------------------------------------------------------------------

def _pred(out: str):
    return [ln.split("|")[-1] for ln in out.splitlines() if "🔶 Pred" in ln]


def _cli(exe, args):
    r = subprocess.run([os.path.join(ROOT, exe)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    return r.returncode, r.stdout


def test_both_stacks_same_greedy_tokens_q80(tmp_models):
    """dllama and dllama-native with --kv-cache-float-type q80: the same greedy tokens (tensor-core prefill, then decode)."""
    m, t = tmp_models["tiny-llama31"]
    common = ["inference", "--model", m, "--tokenizer", t, "--buffer-float-type", "q80", "--prompt", "Hello world, the model " * 6,
              "--steps", "48", "--temperature", "0", "--kv-cache-float-type", "q80"]
    outs = []
    for exe in ("dllama-native", "dllama"):
        rc, out = _cli(exe, common)
        assert rc == 0, out[-2000:]
        outs.append(_pred(out))
    assert len(outs[0]) >= 8 and outs[0] == outs[1]


def test_unknown_kv_cache_type_is_a_one_line_error(tmp_models):
    m, t = tmp_models["tiny-llama31"]
    for exe in ("dllama-native", "dllama"):
        rc, out = _cli(exe, ["inference", "--model", m, "--tokenizer", t, "--prompt", "Hi", "--steps", "4", "--kv-cache-float-type", "fp8"])
        assert rc != 0
        assert "Invalid KV-cache float type: fp8" in out, out[-2000:]


def test_tensor_parallel_q80_equals_one_gpu(tmp_models):
    """dllama-native --gpus 2 on q80 caches: the greedy tokens of one GPU (the short prompt stays on the bit-exact GEMV path)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    m, t = tmp_models["tiny-llama31"]
    common = ["inference", "--model", m, "--tokenizer", t, "--prompt", "Hello world", "--steps", "48", "--temperature", "0",
              "--kv-cache-float-type", "q80"]
    rc1, one = _cli("dllama-native", common)
    rc2, two = _cli("dllama-native", common + ["--gpus", "2"])
    assert rc1 == 0 and rc2 == 0, (one[-1000:], two[-1000:])
    assert len(_pred(one)) >= 8 and _pred(one) == _pred(two)


@pytest.mark.parametrize("server", ["python", "native"])
def test_api_parallel_q80_end_to_end(tmp_models, server):
    """--parallel 4 on q80 caches: four concurrent greedy requests return the text each returns alone."""
    import http.client
    import json
    import socket
    import threading
    import time
    m, t = tmp_models["tiny-llama31"]
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()

    def post(body):
        c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
        try:
            c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
            return json.loads(c.getresponse().read())["choices"][0]["message"]["content"]
        finally:
            c.close()

    cmd = ([sys.executable, "-m", "distributed_llama_b200.apps.api_server"] if server == "python"
           else [os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")])
    proc = subprocess.Popen(cmd + ["--model", m, "--tokenizer", t, "--port", str(port), "--host", "127.0.0.1", "--parallel", "4",
                                   "--temperature", "0", "--kv-cache-float-type", "q80"], cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT),
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.5).close()
                break
            except OSError:
                assert proc.poll() is None, proc.stdout.read()
                time.sleep(0.2)
        bodies = [{"messages": [{"role": "user", "content": f"question number {i} " * (i + 1)}], "max_tokens": 24, "temperature": 0}
                  for i in range(4)]
        alone = [post(b) for b in bodies]
        together = [None] * 4

        def go(i):
            together[i] = post(bodies[i])
        ths = [threading.Thread(target=go, args=(i,)) for i in range(4)]
        for th in ths:
            th.start()
        for th in ths:
            th.join(timeout=120)
        assert together == alone
        assert all(a for a in alone)
    finally:
        proc.kill()
        proc.communicate()
