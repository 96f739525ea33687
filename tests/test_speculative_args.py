"""`--draft-model` / `--draft-tokens` (greedy speculative decoding): flag parsing and every startup refusal of the Python front ends,
without a GPU. The refusals that need the model headers (mixture of experts, non-q40 weights, vocabulary sizes) are raised by
InferenceSession before any weight is loaded."""
import os
import subprocess

import pytest

from distributed_llama_b200.api import DraftRefused, InferenceSession, draft_refusal
from distributed_llama_b200.apps import api_server, cli
from distributed_llama_b200.apps.args import parse_args


def test_flags_parse():
    a = parse_args(["inference", "--model", "m", "--draft-model", "d.m", "--draft-tokens", "7"], True)
    assert (a.draft_model, a.draft_tokens) == ("d.m", 7)
    a = parse_args(["--model", "m", "--draft-model", "d.m"], False)
    assert (a.draft_model, a.draft_tokens) == ("d.m", 3)
    assert parse_args(["chat", "--model", "m"], True).draft_model is None


@pytest.mark.parametrize("k,ok", [(1, True), (3, True), (7, True), (0, False), (2, False), (4, False), (8, False)])
def test_draft_tokens_range(k, ok):
    assert (draft_refusal(k) is None) == ok
    if not ok:
        assert draft_refusal(k) == "--draft-tokens must be 1, 3 or 7"


def test_flag_refusals(monkeypatch):
    assert "one GPU" in draft_refusal(3, n_ranks=2)
    assert "--parallel" in draft_refusal(3, parallel=2)
    monkeypatch.setenv("DL_COLLECTIVES", "nccl")
    assert "DL_COLLECTIVES=nccl" in draft_refusal(3)


@pytest.mark.parametrize("extra,needle", [(["--gpus", "2"], "one GPU"), (["--workers", "10.0.0.1:9999"], "one GPU"),
                                          (["--draft-tokens", "5"], "1, 3 or 7")])
def test_cli_refuses_at_startup(capsys, extra, needle):
    rc = cli.main(["inference", "--model", "m.m", "--tokenizer", "t.t", "--prompt", "x", "--steps", "8", "--draft-model", "d.m"] + extra)
    out = capsys.readouterr().out.strip().splitlines()
    assert rc == 1 and len(out) == 1 and out[0].startswith("🚨 Critical error: ") and needle in out[0], out


@pytest.mark.parametrize("extra,needle", [(["--gpus", "2"], "one GPU"), (["--workers", "10.0.0.1:9999"], "one GPU"),
                                          (["--parallel", "2"], "--parallel"), (["--draft-tokens", "0"], "1, 3 or 7")])
def test_api_server_refuses_at_startup(capsys, extra, needle):
    rc = api_server.main(["--model", "m.m", "--tokenizer", "t.t", "--draft-model", "d.m"] + extra)
    err = capsys.readouterr().err.strip().splitlines()
    assert rc == 1 and len(err) == 1 and needle in err[0], err


def test_api_server_refuses_nccl(capsys, monkeypatch):
    monkeypatch.setenv("DL_COLLECTIVES", "nccl")
    assert api_server.main(["--model", "m.m", "--tokenizer", "t.t", "--draft-model", "d.m"]) == 1
    assert "DL_COLLECTIVES=nccl" in capsys.readouterr().err


def test_no_draft_no_refusal(capsys):
    """Without --draft-model a bad --draft-tokens is not looked at (the flag has no effect)."""
    assert api_server.main(["--model", "m.m", "--draft-tokens", "5", "--help"]) == 0


@pytest.mark.parametrize("target,draft,needle", [
    ("tiny-llama31", "tiny-qwen3-moe", "mixture-of-experts"),
    ("tiny-qwen3-moe", "tiny-qwen3", "mixture-of-experts"),
    ("tiny-llama31", "tiny-llama31-f32", "q40 weights"),
    ("tiny-qwen3-f16", "tiny-qwen3", "q40 weights"),
    ("tiny-llama", "tiny-llama-q80", "q40 weights"),
])
def test_session_refuses_models(tmp_models, target, draft, needle):
    with pytest.raises(DraftRefused, match=needle):
        InferenceSession(tmp_models[target][0], tmp_models[target][1], draft_model=tmp_models[draft][0])


def test_session_refuses_parallel_and_k(tmp_models):
    m, t = tmp_models["tiny-llama31"]
    with pytest.raises(DraftRefused, match="--parallel"):
        InferenceSession(m, t, draft_model=m, parallel=2)
    with pytest.raises(DraftRefused, match="1, 3 or 7"):
        InferenceSession(m, t, draft_model=m, draft_tokens=4)


def test_session_refuses_other_vocabulary(tmp_models, tmp_path):
    import dataclasses

    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    path = str(tmp_path / "vocab1024.m")
    write_synthetic_model(path, dataclasses.replace(get_config("tiny-llama31"), vocab_size=1024), seed=3)
    m, t = tmp_models["tiny-llama31"]
    with pytest.raises(DraftRefused, match="vocabulary: 512 tokens against 1024"):
        InferenceSession(m, t, draft_model=path)


def test_session_refuses_shorter_draft_context(tmp_models, tmp_path):
    import dataclasses

    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    path = str(tmp_path / "ctx256.m")
    write_synthetic_model(path, dataclasses.replace(get_config("tiny-llama31"), max_seq_len=256), seed=3)
    m, t = tmp_models["tiny-llama31"]
    with pytest.raises(DraftRefused, match="context of at least 512 tokens: the draft model has 256"):
        InferenceSession(m, t, draft_model=path)
    # the same draft serves the target run with a context of 256
    assert draft_refusal(3, headers=(("target model", _header(m, 256)), ("draft model", _header(path, 256)))) is None


def _header(path, max_seq_len=0):
    from distributed_llama_b200 import host
    return host().load_model_header(path, max_seq_len)


@pytest.mark.parametrize("model,d,n", [("llama-3.3-70b", 128256, 8192), ("qwen3-14b", 151936, 5120)])
def test_verify_logits_plan_at_eight_rows(model, d, n):
    """The fused per-row arg-max cannot hold 8 rows of these logits GEMVs in shared memory (rc 1): the verify step then runs the STORE
    GEMV, which splits the batch, and one arg-max CTA per row (engine.cu, logits mode 3). Both plans are what that path relies on."""
    from distributed_llama_b200 import ops
    assert ops.gemv_q40_plan(0, 5, 8, d, n, num_sms=132, impl="tma").rc == 1
    assert ops.gemv_q40_plan(0, 5, 2, d, n, num_sms=132, impl="tma").rc == 0
    store = ops.gemv_q40_plan(0, 0, 8, d, n, num_sms=132)
    assert store.rc == 0 and store.launches >= 1


NATIVE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_llama_b200")


@pytest.mark.parametrize("extra,needle", [(["--gpus", "2"], "one GPU"), (["--workers", "10.0.0.1:9999"], "one GPU"),
                                          (["--draft-tokens", "2"], "1, 3 or 7")])
def test_native_cli_refuses_at_startup(extra, needle):
    p = subprocess.run([os.path.join(NATIVE, "dllama-native"), "inference", "--model", "m.m", "--tokenizer", "t.t", "--prompt", "x",
                        "--steps", "8", "--draft-model", "d.m"] + extra, capture_output=True, text=True, timeout=60)
    out = p.stdout.strip().splitlines()
    assert p.returncode == 1 and len(out) == 1 and out[0].startswith("🚨 Critical error: ") and needle in out[0], (p.stdout, p.stderr)


@pytest.mark.parametrize("extra,needle", [(["--gpus", "2"], "one GPU"), (["--workers", "10.0.0.1:9999"], "one GPU"),
                                          (["--parallel", "2"], "--parallel"), (["--draft-tokens", "0"], "1, 3 or 7")])
def test_native_api_server_refuses_at_startup(extra, needle):
    p = subprocess.run([os.path.join(NATIVE, "dllama-api-native"), "--model", "m.m", "--tokenizer", "t.t", "--draft-model", "d.m"] + extra,
                       capture_output=True, text=True, timeout=60)
    err = p.stderr.strip().splitlines()
    assert p.returncode == 1 and len(err) == 1 and needle in err[0], (p.stdout, p.stderr)
