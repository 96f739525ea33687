"""Greedy speculative decoding with a draft model (csrc/cuda/speculative.cu, engine.cu: dl_spec_round): the verify step's per-row
fused arg-max, the accept kernel, and whole completions against greedy decoding without a draft.

Drafts: the target file itself (every draft is expected to be accepted), `tiny-llama-kvrep` with another seed for `tiny-llama31`
(the same 512-token llama3 vocabulary, so drafts are often rejected) and a second `tiny-qwen3` with another seed.

The target's tokens come from the batched verify GEMVs instead of the persistent kernel, so where two logits nearly tie the two
paths may pick different tokens (the README's caveat). With a bf16 cache a speculative completion must return exactly the tokens of
the multi-kernel single-token path; against greedy decoding without a draft (the persistent kernel) it may part only at a near-tie,
whose logit gap is checked against the bounds of the existing cross-path tests."""
import pytest
import torch

from distributed_llama_b200.api import InferenceSession, run_choices
from distributed_llama_b200.ops import cuda_lib as cl

pytestmark = pytest.mark.gpu

PROMPT = "The quick brown fox jumps over the lazy dog and then"


@pytest.fixture(scope="module")
def drafts(tmp_models, tmp_path_factory):
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    root = tmp_path_factory.mktemp("drafts")
    out = {}
    for target, name in (("tiny-llama31", "tiny-llama-kvrep"), ("tiny-qwen3", "tiny-qwen3")):
        path = str(root / f"{name}-draft.m")
        write_synthetic_model(path, get_config(name), seed=29)
        out[target] = {"self": tmp_models[target][0], "other": path}
    return out


_SESSIONS = {}


def session(tmp_models, model, kv="bf16", draft=None, k=3, mega=True):
    """A greedy session, cached; mega=False: single-token steps on the multi-kernel path instead of the persistent kernel."""
    key = (model, kv, draft, k, mega)
    if key not in _SESSIONS:
        m, t = tmp_models[model]
        _SESSIONS[key] = InferenceSession(m, t, temperature=0.0, kv_cache_float_type=kv, draft_model=draft, draft_tokens=k)
        if not mega:
            _SESSIONS[key].engine.enable_mega(False)
    return _SESSIONS[key]


def near_tie(sess, prefix, a, b):
    """|logit a - logit b| after `prefix` (prompt + generated tokens) on sess's multi-kernel path."""
    sess.prefill(prefix[:-1], 0)
    lg = sess.forward_logits(prefix[-1], len(prefix) - 1).float()
    return float((lg[a] - lg[b]).abs())


# Two tokens whose logits lie within twice the bound between two decode paths may swap between them: test_persistent_decode_kernel
# bounds the persistent kernel against the multi-kernel path by 2e-3 (bf16 cache), test_gpu_kv_q80 batched against single steps
# by 3e-2 (q80 cache: the paths round the newest K/V row at different points)
TIE = {"bf16": 4e-3, "q80": 6e-2}


def assert_greedy(mk, got, refs, prompt_toks, what, tie):
    """got: a speculative completion; refs: the same request without a draft on the multi-kernel path and on the persistent kernel.
    Each may only part from got where two logits nearly tie (the README's caveat)."""
    for name, want in refs.items():
        if got != want:
            j = next(i for i in range(min(len(got), len(want))) if got[i] != want[i])
            gap = near_tie(mk, prompt_toks + got[:j], got[j], want[j])
            print(f"{what}: parts from the {name} tokens at {j} ({got[j]} against {want[j]}), logit gap {gap:.2e}")
            assert gap < tie, what


def complete(sess, max_tokens=0, stop_at=None, prompt=PROMPT):
    """One greedy completion through run_choices (the API servers' path): the prompt prefilled, then max_tokens tokens (0: to
    the end of the context); stop_at(tokens) ends it like an end-of-sequence token."""
    toks = sess.tokenizer.encode(prompt, True, True)
    sess.prefill(toks[:-1], 0)
    got = []

    def on_token(i, t):
        got.append(t)
        return stop_at is not None and stop_at(got)

    out = run_choices(sess, toks[-1], len(toks) - 1, 1, max_tokens, sess.engine.seq_len, sess.sampler, 0, on_token)
    assert out[0] == got
    return out[0]


# ---- the verify step ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny-llama31", "tiny-qwen3"])
@pytest.mark.parametrize("nb", [2, 4, 8])
def test_verify_rows(tmp_models, model, nb):
    """Per-row logits of the verify forward against nb = 1 multi-kernel steps at the same positions (within 1e-2, as the slots
    test), and each row's arg-max against the host arg-max of that row's logits."""
    sess = session(tmp_models, model)
    eng = sess.engine
    toks = sess.tokenizer.encode(PROMPT, True, True)
    p = len(toks) - 1
    eng.prefill(toks[:-1], 0, want_logits=False)
    rows = [toks[-1]] + [(37 * i + 11) % 500 for i in range(1, nb)]
    arg = eng.verify(rows, p)
    lv = eng.logits[:nb].clone()
    for b in range(nb):
        want = int(torch.argmax(lv[b]))   # lowest index among equal maxima
        assert arg[b] == want, f"row {b}: arg-max {arg[b]}, host {want}"
    eng.enable_mega(False)
    try:
        single = []
        for b in range(nb):
            eng.forward_batch([rows[b]], p + b, logits_mode=1)
            single.append(eng.logits[0].clone())
    finally:
        eng.enable_mega(True)
    ls = torch.stack(single)
    diff = float((lv - ls).abs().max())
    print(f"{model} nb={nb}: verify rows against one-token steps max |diff| {diff:.3g}, bitwise equal {torch.equal(lv, ls)}")
    assert diff < 1e-2


AD, AN = 5000, 2048


@pytest.mark.parametrize("nb", [2, 4, 8])
@pytest.mark.parametrize("limit", [0, AD - 1, 1200])
def test_argmax_rows_crafted(nb, limit):
    """The per-row arg-max epilogue on crafted weights: every row has its maximum tied bitwise with a weight row in another CTA,
    row 0's maximum is planted in the last row of the vocabulary, and the vocabulary limit hides rows at or above it. The logits
    are bitwise those of the STORE launch, the tokens the lowest-index maxima below the limit, and the counter is left at zero."""
    import test_gpu_gemv as G
    from distributed_llama_b200 import ops
    sms = G._device_sms()
    W = G.Q40(AD, AN, 11)
    x, nw, _ = G.inputs(nb, AN, AD, 11)
    probe = G.run_q40(W, x, G.RMS, G.STORE, nw=nw, impl="tma", sms=sms)
    blk = AN // 32
    for b in range(nb):
        m = G.lowest_max(probe[b])
        for r in (AD - 2 - b, 17 + b):                          # far from m: another CTA at any SM count here
            W.raw[r * blk:(r + 1) * blk] = W.raw[m * blk:(m + 1) * blk]
    m0 = G.lowest_max(probe[0])
    sc = W.raw[m0 * blk:(m0 + 1) * blk, :2].clone().view(torch.float16) * 2
    W.raw[(AD - 1) * blk:AD * blk] = W.raw[m0 * blk:(m0 + 1) * blk]
    W.raw[(AD - 1) * blk:AD * blk, :2] = sc.view(torch.uint8)
    W._dev = None
    store = G.run_q40(W, x, G.RMS, G.STORE, nw=nw, impl="tma", sms=sms)
    lim = AD if limit == 0 else limit
    want = [G.lowest_max(store[b][:lim]) for b in range(nb)]
    if limit == 0:
        assert want[0] == AD - 1
    z = dict(device="cuda")
    val = torch.full((nb * sms,), float("nan"), **z)
    idx = torch.full((nb * sms,), -1, dtype=torch.int32, **z)
    counter = torch.zeros(4, dtype=torch.int32, **z)
    tokens = torch.full((8,), -5, dtype=torch.int32, **z)
    for call in range(2):
        out = torch.full((nb, AD), float("nan"), **z)
        ops.gemv_q40_argmax_rows(W.device(), x, norm_w=nw, eps=G.EPS, out=out, arg_val=val, arg_idx=idx, arg_counter=counter,
                                 tokens=tokens, vocab_limit=limit, num_sms=sms)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), store.view(torch.int32)), f"call {call}: logits differ from the STORE launch"
        assert tokens[:nb].tolist() == want and (tokens[nb:] == -5).all(), (call, tokens.tolist(), want)
        assert int(counter[0]) == 0


# ---- the accept kernel ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("case", ["none", "partial", "all"])
def test_accept_kernel(k, case):
    """Accepted count, emitted tokens, both histories, both engines' next (token, position) and the result block."""
    a = {"none": 0, "partial": k // 2 if k > 1 else 0, "all": k}[case]
    p, cap = 100, 256
    g = [300 + 7 * i for i in range(k + 1)]
    d = [g[i] if i < a else 450 + i for i in range(k)]          # d(i+1) == g(i) exactly for i < a
    z = dict(device="cuda", dtype=torch.int32)
    ver = torch.tensor(g + [-3] * (8 - k - 1), **z)
    tt = torch.tensor([55] + d + [-4] * (7 - k), **z)
    tp = torch.tensor([p] + [-6] * 7, **z)
    dt, dp = torch.full((8,), -8, **z), torch.full((8,), -9, **z)
    th, dh = torch.full((cap,), -7, **z), torch.full((cap,), -7, **z)
    res = torch.full((cl.SPEC_RESULT_WORDS,), -1, **z)
    cl.check(cl.lib().dl_spec_accept(ver.data_ptr(), tt.data_ptr(), tp.data_ptr(), th.data_ptr(), cap, dt.data_ptr(), dp.data_ptr(),
                                      dh.data_ptr(), cap, k, res.data_ptr(), cl.stream_ptr()), "spec_accept")
    torch.cuda.synchronize()
    emitted = g[:a + 1]
    H = cl.SPEC_RESULT_HEAD
    r = res.tolist()
    assert r[:H] == [a, a + 1, k, p + a + 1] and r[H:H + a + 1] == emitted and all(v == -1 for v in r[H + a + 1:]), r
    for h in (th, dh):
        h = h.tolist()
        assert h[p + 1:p + a + 2] == emitted and all(v == -7 for i, v in enumerate(h) if not p + 1 <= i <= p + a + 1)
    assert tt.tolist()[0] == g[a] and tt.tolist()[1:k + 1] == d and int(tp[0]) == p + a + 1
    assert int(dt[0]) == g[a] and int(dp[0]) == p + a + 1


# ---- whole completions ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny-llama31", "tiny-qwen3"])
@pytest.mark.parametrize("kv", ["bf16", "q80"])
@pytest.mark.parametrize("draft", ["self", "other"])
@pytest.mark.parametrize("k", [1, 3, 7])
def test_session_tokens(tmp_models, drafts, model, kv, draft, k):
    """Greedy completions with a draft return the tokens of the same completions without one: to the end of the 512-row context,
    max_tokens ending inside a round, an end of sequence inside a round, and a follow-up prefilled after the first answer (the
    prompt cache's reuse)."""
    base = session(tmp_models, model, kv)
    mk = session(tmp_models, model, kv, mega=False)
    spec = session(tmp_models, model, kv, drafts[model][draft], k)
    toks = spec.tokenizer.encode(PROMPT, True, True)
    what = f"{model} {kv} draft={draft} k={k}"
    full, full_mk = complete(base), complete(mk)
    assert len(full) + len(toks) - 1 == spec.engine.seq_len
    st = spec.spec_stats
    r0, d0, a0 = st.rounds, st.drafted, st.accepted
    got = complete(spec)
    rate = (st.accepted - a0) / max(1, st.drafted - d0)
    print(f"{what}: {st.rounds - r0} rounds, acceptance {rate:.3f}")
    refs = {"persistent kernel": full}
    if kv == "bf16":   # the verify rows are the multi-kernel path's arithmetic (test_verify_rows); with q80 its fused append differs
        assert got == full_mk, what
    assert_greedy(mk, got, refs, toks, what + " to the end of the context", TIE[kv])
    if draft == "self":
        assert rate > 0.9
    for n in (1, 2, 5, 10):
        assert complete(spec, max_tokens=n) == full_mk[:n]
    eos = full_mk[6]
    stop = lambda t: t[-1] == eos
    want = full_mk[:full_mk.index(eos) + 1]
    assert complete(mk, stop_at=stop) == want and complete(spec, stop_at=stop) == want
    follow = spec.tokenizer.encode(" and more", False, True)
    outs = []
    for s in (mk, spec):
        complete(s, max_tokens=20)
        P = len(toks) - 1 + 20
        s.prefill(follow[:-1], P)
        outs.append(run_choices(s, follow[-1], P + len(follow) - 1, 1, 16, s.engine.seq_len, s.sampler, 0, lambda i, t: False)[0])
    assert outs[0] == outs[1]


@pytest.mark.parametrize("model", ["tiny-llama31", "tiny-qwen3"])
def test_stop_string_from_accepted_draft(tmp_models, drafts, model):
    """A `stop` string completed by an accepted draft token cuts the text where greedy decoding without a draft cuts it."""
    base = session(tmp_models, model, mega=False)
    spec = session(tmp_models, model, draft=drafts[model]["self"], k=7)
    full = complete(base, max_tokens=40)
    text = "".join(base.tokenizer.decode(t).decode("utf-8", errors="replace") for t in full)
    stop = text[12:18]
    a0 = spec.spec_stats.accepted
    base.reset()
    spec.reset()
    want = base.generate_choices(PROMPT, 1, 40, stop=stop)
    got = spec.generate_choices(PROMPT, 1, 40, stop=stop)
    assert got == want and stop not in got[0] and spec.spec_stats.accepted > a0


@pytest.mark.parametrize("model", ["tiny-llama31", "tiny-qwen3"])
@pytest.mark.parametrize("k", [1, 3, 7])
def test_graph_rounds_equal_eager(tmp_models, drafts, model, k):
    """Rounds replayed from the round graph emit what eager rounds emit, and so does generate() through the session."""
    spec = session(tmp_models, model, draft=drafts[model]["other"], k=k)
    toks = spec.tokenizer.encode(PROMPT, True, True)
    runs = []
    for use_graph in (False, True, True):
        spec.prefill(toks[:-1], 0)
        tok, pos, out = toks[-1], len(toks) - 1, []
        while len(out) < 100:
            emitted, _, _ = spec.engine.spec_round(spec.draft, tok, pos, k, use_graph=use_graph)
            out += emitted
            pos += len(emitted)
            tok = emitted[-1]
        runs.append(out)
    assert runs[0] == runs[1] == runs[2]
    mk = session(tmp_models, model, mega=False)
    spec.reset()
    mk.reset()
    assert spec.generate(PROMPT, 80) == mk.generate(PROMPT, 80)


def test_refused_round_shapes(tmp_models):
    """The C entry refuses a draft of another KV-cache type, the target as its own draft and a draft length outside 1, 3, 7."""
    a = session(tmp_models, "tiny-llama31")
    q = session(tmp_models, "tiny-llama31", "q80")
    import ctypes
    out = (ctypes.c_int32 * cl.SPEC_RESULT_WORDS)()
    L = cl.lib()
    assert L.dl_spec_round(a.engine._h, q.engine._h, 1, 10, 3, 1, out, cl.stream_ptr()) == -72
    assert L.dl_spec_round(a.engine._h, a.engine._h, 1, 10, 3, 1, out, cl.stream_ptr()) == -72
    b = session(tmp_models, "tiny-qwen3")
    assert L.dl_spec_round(a.engine._h, b.engine._h, 1, 10, 4, 1, out, cl.stream_ptr()) == -75


@pytest.mark.parametrize("nb", [2, 8])
@pytest.mark.parametrize("vocab", [1000, 128256])
def test_argmax_rows_kernel(nb, vocab):
    """The per-row arg-max kernel the verify step falls back to when the fused epilogue does not fit (Llama-3.3-70B, Qwen3-14B logits
    at 8 rows): lowest id among equal maxima inside a thread, across warps and at the last id, -inf entries, ids past `vocab`
    (the vocabulary limit) never read."""
    g = torch.Generator(device="cuda").manual_seed(vocab + nb)
    stride = vocab + 64
    lg = torch.randn(nb, stride, device="cuda", generator=g)
    lg[torch.rand(nb, stride, device="cuda", generator=g) < 0.05] = float("-inf")
    lg[:, vocab:] = 1e30                                       # past the limit
    for b in range(nb):
        hi = 50.0 + b
        ties = {0: [vocab - 1], 1: [5, 5 + 1024], 2: [vocab // 2, vocab // 2 + 1]}.get(b % 3, [7])
        if b == nb - 1:
            ties = [vocab - 1]
        lg[b, ties] = hi
    out = torch.full((8,), -5, dtype=torch.int32, device="cuda")
    cl.check(cl.lib().dl_argmax_rows(lg.data_ptr(), stride, vocab, nb, out.data_ptr(), cl.stream_ptr()), "argmax_rows")
    torch.cuda.synchronize()
    want = [int(torch.argmax(lg[b, :vocab])) for b in range(nb)]
    assert out[:nb].tolist() == want and (out[nb:] == -5).all()
