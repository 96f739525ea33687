"""Decode attention of the persistent kernel reads the cached K/V rows from its ring (the producer issues one fill per 64 cached rows of
each attention item this CTA owns, between the layer's QKV and WO fills) and starts without a grid barrier after QKV.

Every step is compared with the fused attention kernel over identical caches. The caches hold random rows, so every position up to
the last row of a 4096-token context is covered: 0, 1 and both sides of every multiple of 64 (the ring's chunk) and of 256 (where the
effective split count grows). The split count, the grid size (16 CTAs: several attention items per CTA, several K/V fills per item)
and the producer pacing are varied; a captured decode graph is replayed across split boundaries."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

SEQ = 4096
POSITIONS = sorted({0, 1, SEQ - 1} | {q for m in range(64, SEQ, 64) for q in (m - 1, m)})
BOUND = 2e-3                     # persistent vs fused: same math, different split boundaries (test_gpu_decode_attn.py)


@pytest.fixture(scope="module")
def long_models(tmp_path_factory):
    """tiny-llama31 (head dim 64, GQA 2) and tiny-qwen3 (head dim 128, GQA 2, QK-norm) with a 4096-token context."""
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    root = tmp_path_factory.mktemp("ring_models")
    out = {}
    for name in ("tiny-llama31", "tiny-qwen3"):
        path = str(root / f"{name}-4k.m")
        write_synthetic_model(path, dataclasses.replace(get_config(name), max_seq_len=SEQ), seed=7, attn_gain=2.0)
        out[name] = path
    return out


def _engine(path, monkeypatch, n_splits=0, ctas=None, inflight=None):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    for var, val in (("DL_MEGA_CTAS", ctas), ("DL_MEGA_INFLIGHT", inflight)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    eng = Engine(load_device_weights(ModelFile(path)), n_splits=n_splits)
    eng.enable_mega(True)            # the environment is read here
    return eng


def _random_caches(eng, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return ([torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.k_cache],
            [torch.randn(c.shape, generator=g, device="cuda").to(c.dtype) for c in eng.v_cache])


def _load(eng, caches):
    for d, s in zip(eng.k_cache + eng.v_cache, caches[0] + caches[1]):
        d.copy_(s)


# (DL_MEGA_CTAS, DL_MEGA_INFLIGHT): the default grid and pacing first
VARIANTS = [(None, None), (None, "2"), (None, "0"), ("16", None), ("16", "2"), ("16", "0")]


@pytest.mark.parametrize("n_splits", [0, 3, 32])
@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_persistent_attention_matches_fused(long_models, monkeypatch, name, n_splits):
    """At every position: the persistent kernel's logits are bitwise equal across grid sizes and producer pacings (an item's math
    does not depend on which CTA runs it or when its fills land), and within BOUND of the fused kernel's. The activations are
    quantised to q80 before every GEMV, so a last-bit difference in attention can move one int8 step of a later activation and
    the logits by ~1e-2: a few positions may exceed BOUND, none by a wrong row, chunk or split (those are off at most positions)."""
    engines = [_engine(long_models[name], monkeypatch, n_splits, ctas, inflight) for ctas, inflight in VARIANTS]
    fused = _engine(long_models[name], monkeypatch, n_splits)
    fused.enable_mega(False)
    caches = _random_caches(fused, 1234 + n_splits)
    errs = {}
    for pos in POSITIONS:
        tok = (7 * pos + 3) % 500 + 1
        _load(fused, caches)
        want = fused.step(tok, pos)
        got = []
        for (ctas, inflight), eng in zip(VARIANTS, engines):
            _load(eng, caches)
            got.append(eng.step(tok, pos).clone())
            assert eng.mega_active, f"the persistent kernel did not run (DL_MEGA_CTAS={ctas})"
            assert torch.equal(got[-1], got[0]), f"pos {pos}: DL_MEGA_CTAS={ctas} DL_MEGA_INFLIGHT={inflight} differs from the default"
        assert bool(torch.isfinite(got[0]).all()), f"pos {pos}: non-finite logits"
        errs[pos] = (got[0] - want).abs().max().item()
    over = {p: e for p, e in errs.items() if e >= BOUND}
    assert len(over) <= len(POSITIONS) // 32, f"persistent vs fused beyond {BOUND} at {len(over)} positions: {over}"
    assert max(errs.values()) < 0.05, over


@pytest.mark.parametrize("ctas", [None, "16"])
@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_persistent_graph_replay_across_splits(long_models, monkeypatch, name, ctas):
    """One captured graph replayed from positions whose steps cross the 64-row chunk and 256-position split boundaries (the
    producer and the consumers re-derive the split count from the device-resident position at every replay): the greedy tokens
    and the K/V rows the kernel appends equal those of eager launches."""
    eng = _engine(long_models[name], monkeypatch, 0, ctas)
    caches = _random_caches(eng, 99)
    n = 24
    for start in (50, 250, 1010, 2040, SEQ - 1 - n):
        out, rows = {}, {}
        for use_graph in (True, False):
            _load(eng, caches)
            out[use_graph] = eng.decode_greedy(11, start, n, use_graph=use_graph)
            assert eng.mega_active
            rows[use_graph] = [c[:, start:start + n].clone() for c in eng.k_cache + eng.v_cache]
        assert out[True] == out[False], start
        for a, b in zip(rows[True], rows[False]):
            assert torch.equal(a, b), start
