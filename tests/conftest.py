import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def tmp_models(tmp_path_factory):
    """Synthetic tiny model files shared by the test session: name -> (model path, tokenizer path)."""
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model, write_synthetic_tokenizer

    root = tmp_path_factory.mktemp("models")
    out = {}
    for name in ("tiny-llama", "tiny-llama31", "tiny-qwen3", "tiny-qwen3-moe"):
        cfg = get_config(name)
        m = str(root / f"{name}.m")
        t = str(root / f"{name}.t")
        write_synthetic_model(m, cfg, seed=7)
        write_synthetic_tokenizer(t, cfg.vocab_size, style="chatml" if "qwen" in name else "llama3")
        out[name] = (m, t)
    # non-q40 weight files (dense f32 / f16 kernels; q80 blocks are dequantised at load)
    from distributed_llama_b200.formats import quants
    for name, base, wt in (("tiny-llama31-f32", "tiny-llama31", quants.F_32), ("tiny-qwen3-f16", "tiny-qwen3", quants.F_16),
                           ("tiny-llama-q80", "tiny-llama", quants.F_Q80)):
        m = str(root / f"{name}.m")
        write_synthetic_model(m, get_config(base), weights_float_type=wt, seed=7)
        out[name] = (m, out[base][1])
    return out
