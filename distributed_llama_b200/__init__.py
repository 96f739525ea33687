"""distributed_llama_b200 — a Hopper (H100, sm_90a) native tensor-parallel LLM inference engine with the
capabilities of b4rtaz/distributed-llama: `.m`/`.t` files, q40 weights, q80 activation buffers,
Llama-3.x / Qwen3 / Qwen3-MoE, `dllama inference|chat|perplexity|worker` and `dllama-api`.

Layout
  formats/   .m / .t readers+writers, numpy codecs           (native twin: csrc/host)
  models/    model configs, synthetic generator, PyTorch f32 oracle, device weight loader
  ops/       ctypes bindings of the hand-written sm_90a kernels (csrc/cuda)
  parallel/  one-process-per-GPU bootstrap, peer-memory arena, collectives
  runtime/   engine wrapper (CUDA-graph decode loop), generation drivers
  (tokenizer, sampler, chat templates, stop detector: native only, csrc/host/text.cpp, reached through host())
  apps/      `dllama` CLI and `dllama-api` HTTP server
"""
__version__ = "0.1.0"


def host():
    """The pybind11 host library (built on first use)."""
    from . import _build
    _build.build_host()
    from . import _host  # type: ignore
    return _host
