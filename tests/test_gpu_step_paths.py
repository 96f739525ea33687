"""The library session and the tensor-parallel root draw the same tokens and send the control packets workers expect.

Each scenario runs api.run_choices twice on one GPU from the same prompt: (A) through an InferenceSession and (B) through an
apps.runtime.RootInference over a second session of the same model and seed, with a channel stub that records every packet and
a communicator stub of two ranks (no communicator for logprobs, which run on one rank only: then nothing is sent). A and B must
return the same tokens and logprobs entries, and B's packets must equal the stream written out below: op, position and words,
with the token words taken from the returned tokens.
"""
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# the control ops (apps.runtime.worker_loop)
STOP, PREFILL, STEP_LOGITS, STEP_GREEDY, STEP_SAMPLE, SEED = 0, 1, 2, 3, 5, 6
CHOICES_SEED, CHOICES_FIRST, CHOICES_STEP, CONTROLS, FILTERS = 7, 8, 9, 10, 11

PROMPT = [3, 17, 250, 9, 44]
P = len(PROMPT) - 1
T, TOPP, SEED_VALUE, BASE = 0.8, 0.9, 4242, 99
PENALTIES = dict(presence_penalty=0.75, frequency_penalty=1.5, logit_bias={"7": 4.0, "11": -100.0, "300": 2.5})


def f32(*xs):
    return [int(w) for w in np.array(xs, dtype=np.float32).view(np.int32)]


def seed_words(s):
    return [s & 0x7FFFFFFF, (s >> 31) & 0x7FFFFFFF, (s >> 62) & 0x3]


def controls(row_mask):
    return (CONTROLS, 0, f32(0.75, 1.5) + [row_mask] + [7] + f32(4.0) + [11] + f32(-100.0) + [300] + f32(2.5))


def fed(toks):
    """The token each step of a single sequence feeds: the prompt's last one, then each draw."""
    return [PROMPT[-1]] + toks[:-1]


def greedy_steps(toks):
    return [(STEP_GREEDY, P + j, [t]) for j, t in enumerate(fed(toks))]


def sampled_steps(toks):
    return [(STEP_SAMPLE, P + j, [t] + f32(T, TOPP)) for j, t in enumerate(fed(toks))]


class Chan:
    def __init__(self):
        self.packets = []

    def send(self, op, pos, tokens):
        self.packets.append((op, pos, list(tokens)))

    def close(self):
        pass


def _pair(tmp_models, name, temperature, ranks=2, **settings):
    """(A, B, B's session, B's channel), both with the prompt prefilled."""
    from distributed_llama_b200.api import InferenceSession
    from distributed_llama_b200.apps.runtime import RootInference
    m, t = tmp_models[name]
    a, sb = (InferenceSession(m, t, temperature=temperature, topp=TOPP, seed=SEED_VALUE, **settings) for _ in range(2))
    chan = Chan()
    b = RootInference(sb, SimpleNamespace(rank=0, world_size=2) if ranks == 2 else None, chan)
    a.prefill(PROMPT[:-1])
    b.prefill(PROMPT[:-1], 0)
    return a, b, sb, chan


def _run(backend, sess, n, max_tokens, stop=None, logprobs=None):
    """run_choices from the prompt's end; stop = {choice: its last token's number}. Returns (tokens, logprobs entries)."""
    from distributed_llama_b200.api import run_choices
    counts, entries = [0] * n, [[] for _ in range(n)]

    def on_token(i, tok):
        counts[i] += 1
        return (stop or {}).get(i) == counts[i]
    lp = {} if logprobs is None else dict(logprobs=logprobs, on_logprobs=lambda i, e: entries[i].append(e))
    out = run_choices(backend, PROMPT[-1], P, n, max_tokens, sess.engine.seq_len, sess.sampler, BASE, on_token, **lp)
    return out, entries


def _both(a, b, sb, n, max_tokens, **kw):
    ta, la = _run(a, a, n, max_tokens, **kw)
    tb, lb = _run(b, sb, n, max_tokens, **kw)
    assert ta == tb
    assert la == lb
    return ta, la


def test_greedy(tmp_models):
    a, b, sb, chan = _pair(tmp_models, "tiny-llama31", 0.0)
    (toks,), _ = _both(a, b, sb, 1, 12)
    b.finish()
    assert len(toks) == 12
    assert chan.packets == [(PREFILL, 0, PROMPT[:-1])] + greedy_steps(toks) + [(STOP, 0, [])]


def test_greedy_logprobs(tmp_models):
    a, b, sb, chan = _pair(tmp_models, "tiny-qwen3", 0.0, ranks=1)
    (toks,), (entries,) = _both(a, b, sb, 1, 8, logprobs=3)
    b.finish()
    assert [e[0] for e in entries] == toks and all(len(e[2]) == 3 for e in entries)
    assert chan.packets == []


def test_sampled_with_controls_and_filters(tmp_models):
    a, b, sb, chan = _pair(tmp_models, "tiny-llama31", T, top_k=40, min_p=0.05, **PENALTIES)
    (first,), _ = _both(a, b, sb, 1, 10)
    (second,), _ = _both(a, b, sb, 1, 10)   # a new completion: its counts start from zero, the generator continues
    b.finish()
    assert 11 not in first + second
    assert chan.packets == ([(PREFILL, 0, PROMPT[:-1]), (SEED, 0, seed_words(SEED_VALUE)), controls(1), (FILTERS, 0, [40] + f32(0.05))]
                            + sampled_steps(first) + [controls(1)] + sampled_steps(second) + [(STOP, 0, [])])


def test_batched_choices(tmp_models):
    from distributed_llama_b200 import host
    a, b, sb, chan = _pair(tmp_models, "tiny-llama31", T, **PENALTIES)
    assert b.batched_choices(3)
    out, _ = _both(a, b, sb, 3, 8, stop={1: 4})
    b.finish()
    assert [len(o) for o in out] == [8, 4, 8]
    C = (sb.engine.seq_len - 1 - P) // 3
    seeds = [w for i in range(3) for w in seed_words(host().choice_seed(BASE, i))]
    steps = []
    for j in range(max(len(o) for o in out) - 1):
        mask = sum(1 << i for i, o in enumerate(out) if len(o) > j + 1)
        # a finished choice keeps feeding its last token
        steps.append((CHOICES_STEP, P, [C, j, mask] + f32(T, TOPP) + [o[min(j, len(o) - 1)] for o in out]))
    assert chan.packets == ([(PREFILL, 0, PROMPT[:-1]), (CHOICES_SEED, 0, seeds), controls(0b1110),
                             (CHOICES_FIRST, P, [PROMPT[-1], 3] + f32(T, TOPP))] + steps + [(STOP, 0, [])])


def test_sequential_choices_restore_the_generator(tmp_models):
    """Mixture-of-experts layers have no batched step: each choice re-seeds the single-sequence generator, and the stream the
    completion before them left is restored afterwards."""
    from distributed_llama_b200 import host
    a, b, sb, chan = _pair(tmp_models, "tiny-qwen3-moe", T, **PENALTIES)
    assert not b.batched_choices(3)
    (first,), _ = _both(a, b, sb, 1, 6)
    state = a.engine.sampler_state()
    choices, _ = _both(a, b, sb, 3, 5)
    (last,), _ = _both(a, b, sb, 1, 6)
    b.finish()
    want = [(PREFILL, 0, PROMPT[:-1]), (SEED, 0, seed_words(SEED_VALUE)), controls(1)] + sampled_steps(first)
    for i, toks in enumerate(choices):
        want += [(SEED, 0, seed_words(host().choice_seed(BASE, i))), controls(1)] + sampled_steps(toks)
    want += [(SEED, 0, seed_words(state)), controls(1)] + sampled_steps(last) + [(STOP, 0, [])]
    assert chan.packets == want


def test_host_sampler(tmp_models, monkeypatch):
    """DL_HOST_SAMPLER=1: both draw on the host from logits copied back, and the device generator is never seeded."""
    monkeypatch.setenv("DL_HOST_SAMPLER", "1")
    a, b, sb, chan = _pair(tmp_models, "tiny-llama31", T)
    (toks,), _ = _both(a, b, sb, 1, 10)
    b.finish()
    assert a._dev_seeded is None and b._dev_seeded is None
    assert chan.packets == ([(PREFILL, 0, PROMPT[:-1])] + [(STEP_LOGITS, P + j, [t]) for j, t in enumerate(fed(toks))]
                            + [(STOP, 0, [])])
