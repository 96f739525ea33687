"""Sampling controls on the device (csrc/cuda/sampler.cu, the engine, both choices paths) against the host Sampler.

* sampleKernel with a bias, random per-row counts and both penalties against the host Sampler drawing from the controlled logits
  (tests/test_sampling_controls.py pins the host transform to the formula bit for bit): greedy agrees on every draw, sampled on
  at least 249 of 250 (the exp tolerance of test_gpu_sampler.py); after the draws every active row's counts grew by exactly its
  token and inactive rows are untouched.
* Engine end to end: device-path tokens with controls equal a loop of engine.step logits and the host Sampler.
* Batched choices: each step's draws equal the host Sampler (one per choice, choice_seed generators) applied to the logits rows that
  step produced. Sequential choices (mixture of experts): each choice equals a fresh single-sequence run with the same controls.
* Controls all zero: greedy decoding stays on the fused arg-max and the captured graph.
"""
import json
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CONTROLS = dict(presence_penalty=0.75, frequency_penalty=1.5, logit_bias={"7": 4.0, "11": -100.0, "300": 2.5})


def _host():
    from distributed_llama_b200 import host
    return host()


@pytest.mark.parametrize("V", [32003, 151936])
@pytest.mark.parametrize("T,topp", [(0.0, 0.0), (0.8, 0.0), (0.8, 0.9), (1.3, 0.0), (1.3, 0.9)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_kernel_matches_host_sampler(V, T, topp, with_bias):
    """with_bias=False also samples a vocabulary n = V - 3 narrower than the logits and count rows (the engine's vocabulary limit
    below a padded embedding table) and passes no bias (penalties only)."""
    from distributed_llama_b200.ops import cuda_lib as cl
    lib, H = cl.lib(), _host()
    rs = np.random.RandomState(V + int(T * 10) + int(topp * 100) + with_bias)
    n = V if with_bias else V - 3
    B, launches = 8, 34                                   # 256 draws: every fourth launch leaves two rows out
    presence, frequency = float(np.float32(rs.uniform(-2, 2))), float(np.float32(rs.uniform(-2, 2)))
    bias = np.zeros(V, dtype=np.float32)
    if with_bias:
        bias[rs.choice(V, 100, replace=False)] = rs.uniform(-100, 100, 100).astype(np.float32)
    counts = np.zeros((B, V), dtype=np.uint32)
    for b in range(B):
        hit = rs.choice(n, 2000, replace=False)
        counts[b, hit] = rs.randint(1, 6, 2000)
    seeds = [int(s) for s in rs.randint(1, 2 ** 62, B)]
    rng = torch.tensor(seeds, dtype=torch.int64, device="cuda")
    hs = [H.Sampler(n, T, topp, s) for s in seeds]        # host generators: the coins of the device rows
    cnt_d = torch.from_numpy(counts.view(np.int32)).cuda()
    bias_d = torch.from_numpy(bias).cuda()
    probs = torch.empty(B * n + 16, device="cuda")
    tok = torch.zeros(B, dtype=torch.int32, device="cuda")
    agree = total = 0
    for k in range(launches):
        mask = 0b00100100 if k % 4 == 3 else 0
        lg = (rs.randn(B, V) * 3).astype(np.float32)
        assert lib.dl_sample_rows_controlled(torch.from_numpy(lg).cuda().data_ptr(), V, probs.data_ptr(), n, T, topp, rng.data_ptr(),
                                             tok.data_ptr(), B, mask, bias_d.data_ptr() if with_bias else None, cnt_d.data_ptr(), V,
                                             presence, frequency, cl.stream_ptr()) == 0
        got = tok.tolist()
        # greedy draws leave the transformed logits in the scratch: the device formula, bit for bit
        scratch = probs[:B * n].view(B, n).cpu().numpy() if T == 0 else None
        for b in range(B):
            if (mask >> b) & 1:
                continue
            x = _controlled(lg[b, :n], counts[b, :n], bias[:n] if with_bias else None, presence, frequency)
            if scratch is not None:
                assert np.array_equal(scratch[b].view(np.uint32), x.view(np.uint32)), (k, b)
            want = int(hs[b].sample(x))                   # no controls on hs: the draw from the controlled logits
            total += 1
            agree += want == got[b]
            counts[b, got[b]] += 1                        # the device counts what it drew
        assert np.array_equal(cnt_d.cpu().numpy().view(np.uint32), counts)
    assert total >= 250
    assert agree == total if T == 0 else agree >= total - 1, (agree, total)


def _controlled(lg, counts, bias, presence, frequency):
    x = lg + bias if bias is not None else lg.copy()
    hit = counts > 0
    x[hit] = (x[hit] - counts[hit].astype(np.float32) * np.float32(frequency)) - np.float32(presence)
    return x


def _session(tmp_models, name, T, seed=4242, **controls):
    from distributed_llama_b200.api import InferenceSession
    m, t = tmp_models[name]
    return InferenceSession(m, t, temperature=T, topp=0.9, seed=seed, **controls)


def _bias_pairs(d):
    return sorted((int(k), float(v)) for k, v in d.items())


PROMPT = [3, 17, 250, 9, 44]


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3", "tiny-qwen3-moe"])
@pytest.mark.parametrize("T", [0.0, 0.8])
def test_engine_controls_match_host_loop(tmp_models, name, T):
    H = _host()
    steps = 24
    dev = _session(tmp_models, name, T, **CONTROLS)
    dev.prefill(PROMPT[:-1])
    dev.sampler.begin_completion()
    tok, got = PROMPT[-1], []
    for _ in range(steps):
        tok = dev.next_token(tok)
        got.append(tok)
    ref = _session(tmp_models, name, T)
    ref.prefill(PROMPT[:-1])
    smp = H.Sampler(ref.sampler.vocab_size, T, 0.9, 4242)
    smp.set_controls(CONTROLS["presence_penalty"], CONTROLS["frequency_penalty"], _bias_pairs(CONTROLS["logit_bias"]))
    tok, want = PROMPT[-1], []
    for _ in range(steps):
        tok = int(smp.sample(ref.forward_logits(tok).float().cpu().numpy()[:smp.vocab_size].copy()))
        want.append(tok)
    assert got == want
    assert 11 not in got                                   # the -100 bias


class _Recorder:
    """Passes every call to the session and keeps the logits rows each batched choices step drew from."""

    def __init__(self, sess):
        self.sess, self.steps = sess, []

    def __getattr__(self, k):
        return getattr(self.sess, k)

    def choices_first(self, token, P, n, T, topp):
        out = self.sess.choices_first(token, P, n, T, topp)
        self.steps.append((self.sess.engine.logits[:1].float().cpu().numpy().copy(), [True] * n, out))
        return out

    def choices_step(self, tokens, P, C, j, active, T, topp):
        out = self.sess.choices_step(tokens, P, C, j, active, T, topp)
        self.steps.append((self.sess.engine.logits[:len(tokens)].float().cpu().numpy().copy(), list(active), out))
        return out


@pytest.mark.parametrize("T", [0.8, 1.3])
def test_batched_choices_match_host_samplers(tmp_models, T):
    from distributed_llama_b200.api import run_choices
    H = _host()
    n, base = 4, 99
    sess = _session(tmp_models, "tiny-llama31", T, **CONTROLS)
    assert sess.batched_choices(n)
    rec = _Recorder(sess)
    sess.prefill(PROMPT[:-1])
    out = run_choices(rec, PROMPT[-1], sess.pos, n, 16, sess.engine.seq_len, sess.sampler, base, lambda i, t: False)
    V = sess.sampler.vocab_size
    hs = []
    for i in range(n):
        s = H.Sampler(V, T, 0.9, H.choice_seed(base, i))
        s.set_controls(CONTROLS["presence_penalty"], CONTROLS["frequency_penalty"], _bias_pairs(CONTROLS["logit_bias"]))
        hs.append(s)
    for k, (lg, active, got) in enumerate(rec.steps):
        for i in range(n):
            if active[i]:
                assert int(hs[i].sample(lg[0 if k == 0 else i][:V].copy())) == got[i], (k, i)
    assert all(len(o) == 16 for o in out) and all(11 not in o for o in out)
    # a second request starts every choice's counts from zero: same seeds, same tokens
    sess2 = _session(tmp_models, "tiny-llama31", T, **CONTROLS)
    sess2.prefill(PROMPT[:-1])
    again = run_choices(sess2, PROMPT[-1], sess2.pos, n, 16, sess2.engine.seq_len, sess2.sampler, base, lambda i, t: False)
    sess.pos = len(PROMPT) - 1
    twice = run_choices(sess, PROMPT[-1], sess.pos, n, 16, sess.engine.seq_len, sess.sampler, base, lambda i, t: False)
    assert again == out and twice == out


def test_sequential_choices_match_single_sequence(tmp_models):
    from distributed_llama_b200.api import run_choices
    H = _host()
    sess = _session(tmp_models, "tiny-qwen3-moe", 0.8, seed=99, **CONTROLS)
    assert not sess.batched_choices(3)
    sess.prefill(PROMPT[:-1])
    got = run_choices(sess, PROMPT[-1], sess.pos, 3, 10, sess.engine.seq_len, sess.sampler, 99, lambda i, t: False)
    for i in range(3):
        s = _session(tmp_models, "tiny-qwen3-moe", 0.8, seed=H.choice_seed(99, i), **CONTROLS)
        s.prefill(PROMPT[:-1])
        s.sampler.begin_completion()
        tok, want = PROMPT[-1], []
        for _ in range(10):
            tok = s.next_token(tok)
            want.append(tok)
        assert got[i] == want, i


def test_zero_controls_keep_the_fused_greedy_path(tmp_models):
    sess = _session(tmp_models, "tiny-llama31", 0.0, presence_penalty=0.0, frequency_penalty=0.0, logit_bias={})
    assert not sess.sampler.controls_active
    sess.prefill(PROMPT[:-1])
    tok, got = PROMPT[-1], []
    for _ in range(12):
        tok = sess.next_token(tok)
        got.append(tok)
    assert sess.engine.graph_captured and sess._dev_controls is None
    ref = _session(tmp_models, "tiny-llama31", 0.0)
    ref.prefill(PROMPT[:-1])
    assert got == ref.engine.decode_greedy(PROMPT[-1], len(PROMPT) - 1, 12)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("T", [0.0, 0.8])
def test_controls_tensor_parallel(tmp_models, tmp_path, T):
    m, t = tmp_models["tiny-llama31"]
    code = f"""
import json, torch
import torch.distributed as dist
from distributed_llama_b200.apps.runtime import init_distributed_from_env, open_control_channel, RootInference, worker_loop
from distributed_llama_b200.api import InferenceSession, run_choices
comm = init_distributed_from_env()
sess = InferenceSession({m!r}, {t!r}, temperature={T}, topp=0.9, seed=7, comm=comm, **{CONTROLS!r})
chan = open_control_channel(comm)
if comm.rank != 0:
    worker_loop(sess, comm, chan)
else:
    inf = RootInference(sess, comm, chan)
    inf.prefill({PROMPT[:-1]!r}, 0)
    out = run_choices(inf, {PROMPT[-1]}, 4, 1, 16, sess.engine.seq_len, sess.sampler, 7, lambda i, t: False)
    inf.finish()
    print("TOKENS " + json.dumps(out[0]))
"""
    script = tmp_path / "tp_controls.py"
    script.write_text(code)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node=2", str(script)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    tp = json.loads(r.stdout.split("TOKENS ")[1].splitlines()[0])
    from distributed_llama_b200.api import run_choices
    one = _session(tmp_models, "tiny-llama31", T, seed=7, **CONTROLS)
    one.prefill(PROMPT[:-1])
    want = run_choices(one, PROMPT[-1], 4, 1, 16, one.engine.seq_len, one.sampler, 7, lambda i, t: False)[0]
    assert tp == want


# ---- the native binaries -------------------------------------------------------------------------------------------------------

ROOT = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
PENALTIES = ["--frequency-penalty", "1.5", "--presence-penalty", "0.5"]


def _native_pred(exe, m, t, extra, gpus=1):
    import os
    argv = [os.path.join(ROOT, exe), "inference", "--model", m, "--tokenizer", t, "--prompt", "Hello world", "--steps", "48"] + extra
    r = subprocess.run(argv + (["--gpus", str(gpus)] if gpus > 1 else []), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    return [ln.split("|")[-1] for ln in r.stdout.splitlines() if "🔶 Pred" in ln]


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_native_cli_controls_match_python_cli(tmp_models, name):
    """Greedy with penalties on one GPU: dllama-native draws with the host Sampler on logits copied back, dllama with sampleKernel's
    arg-max branch on the device. Same tokens; and different from greedy decoding without penalties."""
    m, t = tmp_models[name]
    native = _native_pred("dllama-native", m, t, ["--temperature", "0"] + PENALTIES)
    python = _native_pred("dllama", m, t, ["--temperature", "0", "--buffer-float-type", "q80"] + PENALTIES)
    plain = _native_pred("dllama-native", m, t, ["--temperature", "0"])
    assert len(native) >= 8 and native == python
    assert native != plain


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_native_tensor_parallel_controls(tmp_models):
    """dllama-native --gpus 2 with penalties (TP_OP_CONTROLS, the device sampler on gathered logits) equals one GPU (host Sampler)
    token for token; seeded sampling with penalties under tensor parallelism is reproducible."""
    m, t = tmp_models["tiny-llama31"]
    one = _native_pred("dllama-native", m, t, ["--temperature", "0"] + PENALTIES)
    two = _native_pred("dllama-native", m, t, ["--temperature", "0"] + PENALTIES, gpus=2)
    assert len(one) >= 8 and one == two
    sampled = ["--temperature", "0.8", "--topp", "0.9", "--seed", "4242"] + PENALTIES
    assert _native_pred("dllama-native", m, t, sampled, gpus=2) == _native_pred("dllama-native", m, t, sampled, gpus=2)


def test_native_api_batched_choices_with_controls(tmp_models):
    """dllama-api-native on one GPU, n = 4 sampled choices on the batched device path (TpEngine::choiceControls, count rows 1..4):
    * +100 on one token with frequency and presence penalty 2: every choice opens with a run of at least 20 of that token (each
      choice has its own counts: one shared row would end the runs about four times sooner, near 12) and leaves it before 60
      tokens (the penalty grows with the count);
    * -100 on a token the unbiased request produced: it never appears;
    * a repeated request returns the same choices (counts restart per request); zero controls answer as no controls."""
    import http.client
    import os
    import re
    import socket
    import time
    H = _host()
    m, t = tmp_models["tiny-llama31"]
    tok = H.Tokenizer(t)
    piece = lambda i: bytes(tok.piece(i)).decode("utf-8")
    up = next(i for i in range(tok.vocab_size) if bytes(tok.piece(i)) == "Ġtok7".encode())
    base = {"messages": [{"role": "user", "content": "Hello there"}], "n": 4, "seed": 5, "temperature": 0.8, "max_tokens": 60}
    bodies = [base, dict(base, presence_penalty=0, frequency_penalty=0, logit_bias={}),
              dict(base, logit_bias={str(up): 100}, frequency_penalty=2, presence_penalty=2),
              dict(base, logit_bias={str(up): 100}, frequency_penalty=2, presence_penalty=2)]
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    proc = subprocess.Popen([os.path.join(ROOT, "dllama-api-native"), "--model", m, "--tokenizer", t, "--host", "127.0.0.1", "--port", str(port),
                             "--max-requests", "6", "--temperature", "0"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)

    def post(body):
        c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
        c.request("POST", "/v1/chat/completions", body=json.dumps(body), headers={"Content-Type": "application/json"})
        r = c.getresponse()
        assert r.status == 200
        return [ch["message"]["content"] for ch in json.loads(r.read().decode("utf-8"))["choices"]]

    try:
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.2).close()      # uses one request slot
                break
            except OSError:
                time.sleep(0.1)
        plain, zero, runs, runs_again = [post(b) for b in bodies]
        assert zero == plain and len(set(plain)) > 1
        assert runs == runs_again
        p = piece(up)
        for text in runs:
            k = len(re.match(f"(?:{re.escape(p)}(?!\\d))*", text).group(0)) // len(p)
            assert 20 <= k < 60, (k, text[:200])
        # a filler token the unbiased choices produced (its piece not followed by a digit), banned
        seen = [int(x) for x in re.findall("Ġtok(\\d+)(?!\\d)", "".join(plain))]
        assert seen
        banned = next(i for i in range(tok.vocab_size) if bytes(tok.piece(i)) == f"Ġtok{seen[0]}".encode())
        out = post(dict(base, logit_bias={str(banned): -100}))
        assert not any(re.search(f"Ġtok{seen[0]}(?!\\d)", x) for x in out)
    finally:
        try:
            proc.communicate(timeout=20)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.communicate()
