"""Several completions of one prompt ("choices", csrc/cuda/attn_decode.cu and the engine's choices step).

* choiceAttnKernel (+ ropeKvKernel with a row stride) against a float64 reference over the same bf16 cache. The inputs give
  scores with a standard deviation of about 4, and "needle" keys parallel to choice 0's first q-head sit on the first and last
  prompt rows and on both sides of every prefix split boundary, so a lost or misweighted split moves the output far beyond
  the bound. Tolerance: both sides read the same bf16 cache, so the difference is the kernel's f32 arithmetic (fast exp, online
  softmax rescaling, split merge): 2e-4 * max|V|, the bound tests/test_gpu_decode_attn.py uses for the single-sequence kernels.
  A needle parallel to choice 0's q in choice 1's rows would take choice 0's softmax if choice 0 read those rows.
* The engine's choices step, teacher-forced, against OracleModel at the tolerance of test_engine_matches_oracle.
* Batched draws against the host Sampler with choice_seed generators; the session-level helper; the sequential fallback.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SEQ = 4096
TOL_V = 2e-4
NEEDLE_SCORE = 30.0
EPS = 1e-6
N_SPLITS = 8


def _rope_table(hd: int) -> torch.Tensor:
    import dataclasses
    from distributed_llama_b200 import host
    from distributed_llama_b200.formats import quants
    from distributed_llama_b200.formats.model_file import HEADER_KEYS
    from distributed_llama_b200.models.config import get_config
    cfg = dataclasses.replace(get_config("tiny-qwen3"), head_dim=hd, max_seq_len=SEQ, rope_theta=10000)
    H = host()
    hdr = H.parse_model_header(H.build_model_header([(HEADER_KEYS[k], v) for k, v in cfg.header_params(quants.F_Q40).items()]), 0, 0)
    return torch.from_numpy(np.asarray(H.build_rope_table(hdr, SEQ)).copy())


def _norm_rope(x, w, cs):
    x = x.double()
    if w is not None:
        x = w.double() * (x * torch.rsqrt(x.pow(2).mean(dim=-1, keepdim=True) + EPS))
    c, s = cs[..., 0].double(), cs[..., 1].double()
    a, b = x[..., 0::2], x[..., 1::2]
    out = torch.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = a * s + b * c
    return out


def _split_bounds(P: int):
    n_pos = P + 1
    eff = max(1, min(N_SPLITS, (n_pos + 63) // 64))
    chunk = (n_pos + eff - 1) // eff
    return [s * chunk for s in range(1, eff) if s * chunk < n_pos]


@pytest.mark.parametrize("hd,kv_mul", [(64, 1), (128, 4), (64, 4), (128, 1)])
@pytest.mark.parametrize("B", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("P", [0, 63, 64, 300, 2047])
@pytest.mark.parametrize("j", [0, 1, 17])
def test_choice_attention_matches_float64(P, B, hd, kv_mul, j):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    g = torch.Generator().manual_seed(P * 131 + B * 17 + hd + kv_mul * 3 + j)
    n_kv = 2
    n_heads = n_kv * kv_mul
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    qkv_dim = q_dim + 2 * kv_dim
    C = 24
    qk_norm = kv_mul == 4
    cs = _rope_table(hd)
    rope = cs.cuda().contiguous()
    rp = P + 1 + j
    qn = (1.0 + 0.2 * torch.randn(hd, generator=g)) if qk_norm else None
    kn = (1.0 + 0.2 * torch.randn(hd, generator=g)) if qk_norm else None
    qkv = torch.randn(B, qkv_dim, generator=g)
    # the rotated, scaled query rows the kernel will use (float64)
    q = _norm_rope(qkv[:, :q_dim].view(B, n_heads, hd), qn, cs[rp])
    k_new = _norm_rope(qkv[:, q_dim:q_dim + kv_dim].view(B, n_kv, hd), kn, cs[rp])
    v_new = qkv[:, q_dim + kv_dim:].view(B, n_kv, hd)
    scale = 1.0 / math.sqrt(hd)
    # random keys scaled so that the scores q . k / sqrt(hd) have a standard deviation of about 4
    qnorm = q.norm(dim=-1).mean().item()
    kc = (torch.randn(n_kv, SEQ, hd, generator=g) * (4.0 / (qnorm * scale))).bfloat16()
    vc = torch.randn(n_kv, SEQ, hd, generator=g).bfloat16()
    q00 = q[0, 0]                       # choice 0, q-head 0 -> KV head 0
    needle = (q00 / q00.norm() * NEEDLE_SCORE / (q00.norm() * scale)).bfloat16()
    for p in {0, P, *_split_bounds(P), *[b - 1 for b in _split_bounds(P)]}:
        kc[0, p] = needle
    if B > 1 and j > 0:
        kc[0, P + 1 + C] = needle        # choice 1's first own row: choice 0 must not see it
    inactive = (1 << (B - 1)) if B >= 3 else 0
    mask = inactive
    kcd, vcd = kc.cuda(), vc.cuda()
    before_k, before_v = kcd.clone(), vcd.clone()
    qkv_d = qkv.cuda().contiguous()
    pos = torch.full((B,), rp, dtype=torch.int32, device="cuda")
    partial = torch.full((B * n_heads * N_SPLITS * (hd + 2) + 64,), float("nan"), device="cuda")
    counters = torch.zeros(n_kv, dtype=torch.int32, device="cuda")
    out = torch.full((B, q_dim + 16), float("nan"), device="cuda")
    qn_d = qn.float().cuda() if qk_norm else None
    kn_d = kn.float().cuda() if qk_norm else None
    rc = lib.dl_choice_attn(qkv_d.data_ptr(), qkv_dim, pos.data_ptr(), rope.data_ptr(), qn_d.data_ptr() if qk_norm else None,
                            kn_d.data_ptr() if qk_norm else None, EPS, kcd.data_ptr(), vcd.data_ptr(), n_heads, n_kv, hd, SEQ, N_SPLITS,
                            B, P, C, j, mask, partial.data_ptr(), counters.data_ptr(), out.data_ptr(), q_dim + 16, cl.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    kc_after, vc_after = kcd.cpu(), vcd.cpu()
    # rows <= P untouched, counters reset
    assert torch.equal(kc_after[:, :P + 1], before_k[:, :P + 1].cpu()) and torch.equal(vc_after[:, :P + 1], before_v[:, :P + 1].cpu())
    assert int(counters.abs().sum()) == 0
    changed = (kc_after != before_k.cpu()).any(dim=-1).any(dim=0) | (vc_after != before_v.cpu()).any(dim=-1).any(dim=0)
    written = {P + 1 + b * C + j for b in range(B) if not (mask >> b) & 1}
    assert set(torch.nonzero(changed).flatten().tolist()) <= written
    for b in range(B):
        row = P + 1 + b * C + j
        if (mask >> b) & 1:
            assert torch.equal(kc_after[:, row], before_k[:, row].cpu()) and torch.equal(vc_after[:, row], before_v[:, row].cpu())
            continue
        for t, want in ((kc_after[:, row], k_new[b]), (vc_after[:, row], v_new[b].double())):
            err = (t.double() - want).abs()
            ulp = torch.exp2(torch.floor(torch.log2(want.abs().clamp_min(2.0 ** -126))) - 7)
            assert (err <= ulp + 2.0 ** -20 * want.abs().max()).all(), f"choice {b}: K/V row off by more than 1 bf16 ulp"
    # attention reference over the cache as written
    got = out[:, :q_dim].cpu().view(B, n_heads, hd)
    assert torch.isnan(out[:, q_dim:]).all()
    for b in range(B):
        if (mask >> b) & 1:
            continue
        rows = list(range(P + 1)) + list(range(P + 1 + b * C, P + 1 + b * C + j + 1))
        K = kc_after[:, rows].double()
        V = vc_after[:, rows].double()
        s = torch.einsum("kgd,kpd->kgp", q[b].view(n_kv, kv_mul, hd), K) * scale
        ref = torch.einsum("kgp,kpd->kgd", torch.softmax(s, dim=-1), V).reshape(n_heads, hd)
        tol = TOL_V * V.abs().max().item()
        err = (got[b].double() - ref).abs().max().item()
        assert err <= tol, f"choice {b}: max err {err:.3g} > {tol:.3g}"


def test_batched_sampler_matches_host_sampler():
    from distributed_llama_b200 import host
    from distributed_llama_b200.ops import cuda_lib as cl
    lib, H = cl.lib(), host()
    rs = np.random.RandomState(11)
    n, B, seed = 32003, 5, 777
    draws = 250
    for temperature, topp in ((0.8, 0.9), (1.0, 0.0)):
        seeds = [H.choice_seed(seed, i) for i in range(B)]
        rng = torch.tensor([s if s < 2 ** 63 else s - 2 ** 64 for s in seeds], dtype=torch.int64, device="cuda")
        hs = [H.Sampler(n, temperature, topp, s) for s in seeds]
        probs = torch.empty(B * n + 16, device="cuda")
        tok = torch.zeros(B, dtype=torch.int32, device="cuda")
        dev, ref = [[] for _ in range(B)], [[] for _ in range(B)]
        for d in range(draws):
            first = d % 2 == 0           # alternate the one-row and the per-row modes
            lg = (rs.randn(1 if first else B, n) * 3.0).astype(np.float32)
            lgd = torch.from_numpy(lg).cuda()
            assert lib.dl_sample_rows(lgd.data_ptr(), 0 if first else n, probs.data_ptr(), n, temperature, topp, rng.data_ptr(), tok.data_ptr(),
                                      B, 0, cl.stream_ptr()) == 0
            got = tok.tolist()
            for b in range(B):
                dev[b].append(got[b])
                ref[b].append(int(hs[b].sample(lg[0 if first else b].copy())))
        for b in range(B):
            agree = sum(x == y for x, y in zip(dev[b], ref[b]))
            assert agree >= draws - 1, (temperature, topp, b, agree)
    # inactive rows draw nothing and keep their generator
    rng0 = rng.clone()
    tok.fill_(-5)
    assert lib.dl_sample_rows(lgd.data_ptr(), n, probs.data_ptr(), n, 0.8, 0.9, rng.data_ptr(), tok.data_ptr(), B, 0b10110, cl.stream_ptr()) == 0
    t = tok.tolist()
    assert t[1] == t[2] == t[4] == -5 and t[0] >= 0 and t[3] >= 0
    assert torch.equal(rng[[1, 2, 4]], rng0[[1, 2, 4]]) and not torch.equal(rng[[0, 3]], rng0[[0, 3]])


def _engine(tmp_models, name):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    from distributed_llama_b200.runtime import Engine
    mf = ModelFile(tmp_models[name][0])
    return Engine(load_device_weights(mf)), OracleModel(mf, act_quant="q80", device="cuda")


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
@pytest.mark.parametrize("plen", [5, 45])
def test_choices_step_matches_oracle(tmp_models, name, plen):
    eng, oracle = _engine(tmp_models, name)
    rs = np.random.RandomState(plen)
    prompt = [int(x) for x in rs.randint(3, 500, size=plen)]
    P = plen - 1
    n, steps = 3, 6
    forced = [[int(x) for x in rs.randint(3, 500, size=steps)] for _ in range(n)]
    C = (eng.seq_len - 1 - P) // n
    eng.prefill(prompt[:-1], 0, want_logits=False)
    eng.forward_batch([prompt[-1]], P, logits_mode=1)
    refs = [oracle.forward(prompt + forced[b], 0) for b in range(n)]
    assert (eng.logits[0] - refs[0][P]).abs().max().item() < 0.06
    for j in range(steps):
        eng.choices_forward([forced[b][j] for b in range(n)], P, C, j)
        lg = eng.logits[:n].clone()
        for b in range(n):
            err = (lg[b] - refs[b][P + 1 + j]).abs().max().item()
            assert err < 0.06, f"choice {b} step {j}: {err}"
    # the prompt rows are intact: a single-sequence step at P + 1 equals the same step on a fresh engine
    a = eng.step(forced[0][0], P + 1).clone()
    fresh, _ = _engine(tmp_models, name)
    fresh.prefill(prompt[:-1], 0, want_logits=False)
    fresh.forward_batch([prompt[-1]], P, logits_mode=1)
    b = fresh.step(forced[0][0], P + 1)
    assert torch.equal(a, b)


def _session(tmp_models, name, temperature, seed=4242):
    from distributed_llama_b200.api import InferenceSession
    m, t = tmp_models[name]
    return InferenceSession(m, t, temperature=temperature, topp=0.9, seed=seed)


def _token_choices(sess, prompt, n, max_tokens):
    from distributed_llama_b200.api import run_choices
    sess.prefill(prompt[:-1])
    P = sess.pos
    return run_choices(sess, prompt[-1], P, n, max_tokens, sess.engine.seq_len, sess.sampler, sess.sampler.seed, lambda i, t: False)


def test_session_choices(tmp_models):
    prompt = [3, 17, 250, 9, 44]
    a = _token_choices(_session(tmp_models, "tiny-llama31", 0.8), prompt, 4, 12)
    b = _token_choices(_session(tmp_models, "tiny-llama31", 0.8), prompt, 4, 12)
    assert a == b and all(len(c) == 12 for c in a)
    assert len({tuple(c) for c in a}) > 1
    one = _token_choices(_session(tmp_models, "tiny-llama31", 0.8), prompt, 1, 12)
    assert one[0][0] == a[0][0]
    g1 = _token_choices(_session(tmp_models, "tiny-llama31", 0.0), prompt, 1, 10)
    g3 = _token_choices(_session(tmp_models, "tiny-llama31", 0.0), prompt, 3, 10)
    assert g3 == [g1[0]] * 3
    texts = _session(tmp_models, "tiny-llama31", 0.8).generate_choices("hello world", 3, 8)
    assert len(texts) == 3 and all(isinstance(x, str) for x in texts)


def test_choices_fallback_matches_single_sequence(tmp_models):
    from distributed_llama_b200 import host
    H = host()
    prompt = [3, 17, 250, 9, 44]
    sess = _session(tmp_models, "tiny-qwen3-moe", 0.8, seed=99)
    assert not sess.batched_choices(2)
    got = _token_choices(sess, prompt, 2, 10)
    for i in range(2):
        s = _session(tmp_models, "tiny-qwen3-moe", 0.8, seed=H.choice_seed(99, i))
        s.prefill(prompt[:-1])
        tok, want = prompt[-1], []
        for _ in range(10):
            tok = s.next_token(tok)
            want.append(tok)
        assert got[i] == want


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_choices_tensor_parallel(tmp_models, tmp_path):
    import subprocess
    import sys
    m, t = tmp_models["tiny-llama31"]
    code = f"""
import os, torch
from distributed_llama_b200.apps.runtime import init_distributed_from_env
from distributed_llama_b200.api import InferenceSession, run_choices
from distributed_llama_b200.models.reference import OracleModel
from distributed_llama_b200.formats import ModelFile
comm = init_distributed_from_env()
sess = InferenceSession({m!r}, {t!r}, temperature=0.8, topp=0.9, seed=7, comm=comm)
eng = sess.engine
prompt = [3, 17, 250, 9, 44]
P = 4
forced = [[11, 12, 13], [21, 22, 23], [31, 32, 33]]
C = (eng.seq_len - 1 - P) // 3
eng.prefill(prompt[:-1], 0, want_logits=False)
eng.forward_batch([prompt[-1]], P, logits_mode=1)
oracle = OracleModel(ModelFile({m!r}), act_quant="q80", device="cuda")
for j in range(3):
    eng.choices_forward([forced[b][j] for b in range(3)], P, C, j)
    lg = eng._full_logits(eng.logits[:3])
    for b in range(3):
        ref = oracle.forward(prompt + forced[b], 0)[P + 1 + j]
        assert (lg[b] - ref).abs().max().item() < 0.06
out = run_choices(sess, prompt[-1], P, 3, 8, eng.seq_len, sess.sampler, 7, lambda i, t: False)
import torch.distributed as dist
allv = [None, None]
dist.all_gather_object(allv, out)
assert allv[0] == allv[1]
"""
    script = tmp_path / "tp_choices.py"
    script.write_text(code)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node=2", str(script)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
