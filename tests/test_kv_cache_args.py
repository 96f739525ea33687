"""`--kv-cache-float-type` on the command line (CPU only): parsing, refusal of unknown values, the per-rank cache bytes."""
import pytest

from distributed_llama_b200.apps.args import parse_args


def test_default_is_bf16():
    assert parse_args(["inference", "--model", "m"], True).kv_cache_float_type == "bf16"


@pytest.mark.parametrize("value", ["bf16", "q80"])
def test_accepted_values(value):
    assert parse_args(["chat", "--kv-cache-float-type", value], True).kv_cache_float_type == value
    assert parse_args(["--kv-cache-float-type", value, "--parallel", "4"], False).kv_cache_float_type == value


@pytest.mark.parametrize("value", ["f16", "q40", "fp8", "Q80", ""])
def test_unknown_value_is_refused(value):
    with pytest.raises(ValueError, match="Invalid KV-cache float type"):
        parse_args(["inference", "--kv-cache-float-type", value], True)


def test_missing_value_is_refused():
    with pytest.raises(ValueError, match="Missing value"):
        parse_args(["inference", "--kv-cache-float-type"], True)


def test_cache_bytes_by_type():
    from types import SimpleNamespace

    from distributed_llama_b200.apps.runtime import kv_cache_bytes
    # Llama-3.3-70B at its 131072-token context on one rank: 42.9 GB of bf16 K/V, 22.8 GB in q80
    h = SimpleNamespace(n_kv_heads=8, n_layers=80, seq_len=131072, head_dim=128)
    assert kv_cache_bytes(h, 1, "bf16") == 2 * 80 * 131072 * 8 * 128 * 2
    assert abs(kv_cache_bytes(h, 1, "bf16") / 1e9 - 42.9) < 0.05
    assert abs(kv_cache_bytes(h, 1, "q80") / 1e9 - 22.8) < 0.05
    assert kv_cache_bytes(h, 2, "q80") * 2 == kv_cache_bytes(h, 1, "q80")   # KV heads split over the ranks
    assert kv_cache_bytes(h, 16, "q80") == kv_cache_bytes(h, 8, "q80")      # more ranks than KV heads: one replicated head each
