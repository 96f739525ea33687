"""`--draft-model` in the four front ends: both API servers (`dllama-api`, `dllama-api-native`) and both CLIs (`dllama`,
`dllama-native`), each with and without a draft model, must answer the same requests with the same bytes (the Python and native servers with
the same JSON documents).

The requests run in one order on every server, so the prompt cache holds the same conversation everywhere: a greedy non-stream
request, the same request streamed, a multi-turn follow-up that continues the first answer from the prompt cache (both engines
prefill only the new messages), a seeded sampled request and an `n` = 2 request (these two take the single-step path). tiny-qwen3
is used because its greedy tokens on the multi-row verify path and on the persistent kernel agree over these lengths (tiny-llama31's
first near-tie is checked in test_gpu_speculative.py). Only the `created` timestamps are normalised."""
import json
import os
import re
import socket
import subprocess
import sys
import time

import pytest

from test_gpu_stop_sequences import ROOT, Server, _free_port   # noqa: F401

pytestmark = pytest.mark.gpu

MODEL = "tiny-qwen3"
MSGS = [{"role": "user", "content": "write something long"}]


@pytest.fixture(scope="module")
def other_draft(tmp_path_factory):
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    path = str(tmp_path_factory.mktemp("srv-draft") / "qwen3-draft.m")
    write_synthetic_model(path, get_config(MODEL), seed=29)
    return path


class DraftServer(Server):
    """test_gpu_stop_sequences.Server (greedy by default, one slot) with extra flags."""

    def __init__(self, kind, model, extra):
        m, t = model
        self.port = _free_port()
        cmd = ([sys.executable, "-m", "distributed_llama_b200.apps.api_server"] if kind == "python"
               else [os.path.join(ROOT, "distributed_llama_b200", "dllama-api-native")])
        self.proc = subprocess.Popen(cmd + ["--model", m, "--tokenizer", t, "--port", str(self.port), "--host", "127.0.0.1",
                                            "--temperature", "0"] + extra, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT),
                                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, errors="replace")
        for _ in range(600):
            try:
                socket.create_connection(("127.0.0.1", self.port), timeout=0.5).close()
                return
            except OSError:
                assert self.proc.poll() is None, self.proc.stdout.read()
                time.sleep(0.2)


def _norm(raw: bytes) -> bytes:
    return re.sub(rb'"created": ?\d+', b'"created": 0', raw)


def _session(srv):
    out = []
    first = srv.post({"messages": MSGS, "temperature": 0, "max_tokens": 24})
    out.append(first)
    out.append(srv.post({"messages": MSGS, "temperature": 0, "max_tokens": 24, "stream": True}))
    answer = json.loads(first)["choices"][0]["message"]["content"]
    follow = MSGS + [{"role": "assistant", "content": answer}, {"role": "user", "content": "and more"}]
    out.append(srv.post({"messages": follow, "temperature": 0, "max_tokens": 24}))
    out.append(srv.post({"messages": MSGS, "temperature": 0.8, "seed": 7, "max_tokens": 16}))
    out.append(srv.post({"messages": MSGS, "temperature": 0.8, "seed": 3, "n": 2, "max_tokens": 8}))
    return [_norm(r) for r in out]


def test_servers_answer_alike(tmp_models, other_draft):
    model = tmp_models[MODEL]
    runs = {}
    for kind in ("python", "native"):
        for name, extra in (("none", []), ("self", ["--draft-model", model[0], "--draft-tokens", "7"]),
                            ("other", ["--draft-model", other_draft, "--draft-tokens", "3"])):
            srv = DraftServer(kind, model, extra)
            try:
                runs[(kind, name)] = _session(srv)
            finally:
                srv.close()
    for kind in ("python", "native"):   # with and without a draft: the same bytes
        ref = runs[(kind, "none")]
        assert len(ref) == 5 and all(r.startswith(b"{") or r.startswith(b"data:") for r in ref)
        for name in ("self", "other"):
            for i, (a, b) in enumerate(zip(ref, runs[(kind, name)])):
                assert a == b, f"{kind} draft={name} request {i}:\n{a[:400]}\n{b[:400]}"
    # Python and native servers: the same documents (the Python server escapes non-ASCII characters, the native one does not)
    for i, (a, b) in enumerate(zip(runs[("python", "none")], runs[("native", "none")])):
        assert _parsed(a) == _parsed(b), f"python against native, request {i}"


def _parsed(raw: bytes):
    if raw.startswith(b"{"):
        return json.loads(raw)
    return [json.loads(ln[5:]) for ln in raw.split(b"\n") if ln.startswith(b"data:") and ln.strip() != b"data: [DONE]"]


def _cli_pieces(cmd):
    p = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, errors="replace", timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    pieces = [ln.split(" | ", 2)[2] for ln in p.stdout.splitlines() if ln.startswith("🔶 Pred")]
    stats = [ln for ln in p.stdout.splitlines() if ln.startswith("Speculative: ")]
    return pieces, stats


@pytest.mark.parametrize("kind", ["python", "native"])
def test_cli_inference_alike(tmp_models, other_draft, kind):
    """`dllama inference` / `dllama-native inference` print the same tokens with a draft, plus one summary line of the rounds."""
    m, t = tmp_models[MODEL]
    cmd = ([sys.executable, "-m", "distributed_llama_b200.apps.cli"] if kind == "python"
           else [os.path.join(ROOT, "distributed_llama_b200", "dllama-native")])
    cmd += ["inference", "--model", m, "--tokenizer", t, "--prompt", "hello there", "--steps", "48", "--temperature", "0"]
    base, none = _cli_pieces(cmd)
    assert none == [] and len(base) > 30
    for draft, k in ((m, "7"), (other_draft, "1")):
        pieces, stats = _cli_pieces(cmd + ["--draft-model", draft, "--draft-tokens", k])
        assert pieces == base and len(stats) == 1, (draft, k, stats)
        rounds = int(stats[0].split()[1])
        assert 0 < rounds <= len(base)
        if draft == m:
            assert rounds < len(base) / 2, stats[0]   # the target as its own draft: most drafts accepted
