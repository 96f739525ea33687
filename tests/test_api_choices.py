"""`n` completions in the Python API server (CPU): request parsing, response shapes, streaming and the prompt cache, with an
inference stub whose next token depends on the sampler's seed, so that the choices differ."""
import json
import types

import pytest

from distributed_llama_b200 import host
from distributed_llama_b200.apps.api_server import ApiServer, HttpRequest


class StubInference:
    """Single-sequence stub: every call is recorded; next_token mixes a coin of the sampler's generator with (position, token)."""

    def __init__(self, vocab_low: int, vocab_span: int):
        self.low, self.span = vocab_low, vocab_span
        self.prefills, self.steps = [], []

    def prefill(self, tokens, pos):
        if tokens:
            self.prefills.append((list(tokens), pos))

    def next_token(self, token, pos, sampler):
        # draws from the sampler's advancing generator, like the device sampler's stream
        self.steps.append(pos)
        return self.low + (int(sampler.next_coin() * 65536) + pos * 40503 + token * 97) % self.span

    next_token_at = next_token

    def forget_device_seed(self):
        pass

    def save_sampler(self):
        return None

    def restore_sampler(self, saved):
        pass

    def batched_choices(self, n):
        return False


class FakeConn:
    def __init__(self):
        self.data = b""

    def sendall(self, b):
        self.data += b


def _server(tmp_path):
    from distributed_llama_b200.models.synthetic import write_synthetic_tokenizer
    H = host()
    path = str(tmp_path / "tok.t")
    write_synthetic_tokenizer(path, 512, style="llama3")
    tok = H.Tokenizer(path)
    args = types.SimpleNamespace(temperature=0.8, topp=0.9, chat_template="llama3", model="m.m")
    header = types.SimpleNamespace(seq_len=512)
    inf = StubInference(260, 200)   # merged regular tokens: no special token, no end of sequence
    ctx = types.SimpleNamespace(args=args, tokenizer=tok, inference=inf, header=header, sampler=H.Sampler(tok.vocab_size, 0.8, 0.9, 5),
                                sess=None)
    return ApiServer(ctx), inf


def _post(api, body):
    req = HttpRequest(FakeConn())
    req.json = body
    api.complete(req)
    raw = req.conn.data.decode("utf-8")
    head, payload = raw.split("\r\n\r\n", 1)
    if "text/event-stream" in head:
        events = [ln for ln in payload.split("\r\n") if ln.startswith("data: ")]
        return events
    return json.loads(payload)


MSGS = [{"role": "user", "content": "Hello there"}]


def test_non_stream_choices(tmp_path):
    api, inf = _server(tmp_path)
    r = _post(api, {"messages": MSGS, "max_tokens": 7, "n": 3, "seed": 11})
    assert [c["index"] for c in r["choices"]] == [0, 1, 2]
    assert all(c["finish_reason"] == "stop" and c["message"]["role"] == "assistant" for c in r["choices"])
    texts = [c["message"]["content"] for c in r["choices"]]
    assert len(set(texts)) == 3
    assert r["usage"]["completion_tokens"] == 21 and r["usage"]["total_tokens"] == r["usage"]["prompt_tokens"] + 21
    # the same request again gives the same choices
    api2, _ = _server(tmp_path)
    assert _post(api2, {"messages": MSGS, "max_tokens": 7, "n": 3, "seed": 11})["choices"] == r["choices"]
    # choice 0 is what an n-less request with the same seed returns
    api3, _ = _server(tmp_path)
    single = _post(api3, {"messages": MSGS, "max_tokens": 7, "seed": 11})
    assert len(single["choices"]) == 1 and single["choices"][0]["index"] == 0
    assert single["choices"][0]["message"]["content"] == texts[0] and single["usage"]["completion_tokens"] == 7


def test_stream_choices(tmp_path):
    api, _ = _server(tmp_path)
    events = _post(api, {"messages": MSGS, "max_tokens": 5, "n": 3, "stream": True, "seed": 11})
    assert events[-1] == "data: [DONE]" and events.count("data: [DONE]") == 1
    chunks = [json.loads(e[6:]) for e in events[:-1]]
    stops = [c["choices"][0]["index"] for c in chunks if c["choices"][0]["finish_reason"] == "stop"]
    assert stops == [0, 1, 2]
    text = {i: "".join(c["choices"][0]["delta"]["content"] for c in chunks
                       if c["choices"][0]["index"] == i and "delta" in c["choices"][0]) for i in range(3)}
    api2, _ = _server(tmp_path)
    r = _post(api2, {"messages": MSGS, "max_tokens": 5, "n": 3, "seed": 11})
    assert [text[i] for i in range(3)] == [c["message"]["content"] for c in r["choices"]]


def test_follow_up_reuses_the_prompt(tmp_path):
    api, inf = _server(tmp_path)
    r = _post(api, {"messages": MSGS, "max_tokens": 6, "n": 3, "seed": 3})
    prompt_end = inf.steps[0]
    assert [it[0] for it in api.cache.items] == [prompt_end]
    hist = MSGS + [{"role": "assistant", "content": r["choices"][1]["message"]["content"]}, {"role": "user", "content": "more"}]
    n_pref = len(inf.prefills)
    _post(api, {"messages": hist, "max_tokens": 2})
    assert len(inf.prefills) == n_pref + 1 and inf.prefills[-1][1] == prompt_end


@pytest.mark.parametrize("bad", [0, 9, "x", 2.0, True])
def test_bad_n_is_refused_and_the_server_keeps_serving(tmp_path, bad):
    api, inf = _server(tmp_path)
    with pytest.raises(ValueError):
        _post(api, {"messages": MSGS, "max_tokens": 3, "n": bad})
    assert inf.steps == [] and inf.prefills == []
    assert len(_post(api, {"messages": MSGS, "max_tokens": 3, "n": 2})["choices"]) == 2


def test_choice_seed():
    H = host()
    assert H.choice_seed(12345, 0) == 12345
    assert len({H.choice_seed(12345, i) for i in range(8)}) == 8


def test_seedless_requests_differ_and_keep_the_single_stream(tmp_path):
    api, _ = _server(tmp_path)
    a = _post(api, {"messages": MSGS, "max_tokens": 6, "n": 3})
    b = _post(api, {"messages": MSGS, "max_tokens": 6, "n": 3})
    assert [c["message"]["content"] for c in a["choices"]] != [c["message"]["content"] for c in b["choices"]]
    # an n = 1 request after an n = 3 request continues the generator instead of replaying it
    api2, _ = _server(tmp_path)
    first = _post(api2, {"messages": MSGS, "max_tokens": 6})["choices"][0]["message"]["content"]
    _post(api2, {"messages": MSGS, "max_tokens": 6, "n": 3})
    again = _post(api2, {"messages": MSGS, "max_tokens": 6})["choices"][0]["message"]["content"]
    assert again != first


def test_choices_control_ops_round_trip():
    """The root's choices packets, replayed by worker_loop, make the worker's engine repeat the root's engine calls."""
    from distributed_llama_b200.apps import runtime as rt

    class Eng:
        def __init__(self):
            self.calls = []

        def seed_choice_samplers(self, seeds):
            self.calls.append(("seed", list(seeds)))

        def choices_first(self, token, P, n, T, topp):
            self.calls.append(("first", token, P, n, T, topp))
            return [1] * n

        def choices_step(self, tokens, P, C, j, active, T, topp):
            self.calls.append(("step", list(tokens), P, C, j, list(active), T, topp))
            return list(tokens)

        def supports_choices(self, n):
            return True

    class Chan:
        def __init__(self):
            self.packets = []

        def send(self, op, pos, tokens):
            self.packets.append((op, pos, list(tokens)))

        def recv(self):
            return self.packets.pop(0) if self.packets else (rt.OP_STOP, 0, [])

        def close(self):
            pass

    root_eng, worker_eng, chan = Eng(), Eng(), Chan()
    sess = types.SimpleNamespace(engine=root_eng, header=None, device="cpu")
    root = rt.RootInference(sess, comm=types.SimpleNamespace(world_size=2), chan=chan)
    seeds = [host().choice_seed(2 ** 63 + 12345, i) for i in range(3)]
    root.seed_choices(seeds)
    root.choices_first(77, 40, 3, 0.8, 0.9)
    root.choices_step([5, 6, 7], 40, 100, 2, [True, False, True], 0.8, 0.9)
    rt.worker_loop(types.SimpleNamespace(engine=worker_eng, device="cpu"), None, chan)
    f32 = lambda x: rt._bits_f32(*rt._f32_bits(x))[0]
    assert worker_eng.calls == [c if c[0] == "seed" else tuple(f32(v) if isinstance(v, float) else v for v in c) for c in root_eng.calls]
    assert worker_eng.calls[0] == ("seed", seeds)
