"""Command-line flags of `dllama` / `dllama-api` — same surface as the reference parser (src/app.cpp:24-135):
`--key value` pairs, first positional = mode, `--workers` variadic, `--help/-h/--usage` short-circuit, unknown flags
are an error. Flags that only make sense for the CPU/TCP design (`--nthreads`, `--net-turbo`, `--gpu-index`,
`--gpu-segments`, `--workers host:port`) are accepted for drop-in compatibility; on the GPU build the worker set is
the torch.distributed world (one process per GPU), so `--workers` only has to name as many entries as there are ranks-1.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import List, Optional


@dataclass
class AppArgs:
    mode: Optional[str] = None
    help: bool = False
    info: bool = True
    model: Optional[str] = None
    tokenizer: Optional[str] = None
    prompt: Optional[str] = None
    buffer_float_type: str = "q80"
    workers: List[str] = field(default_factory=list)
    host: str = "0.0.0.0"
    port: int = 9990
    nthreads: int = 1
    n_batches: int = 32
    steps: int = 0
    temperature: float = 0.8
    topp: float = 0.9
    presence_penalty: float = 0.0    # sampling controls (host Sampler.set_controls), each in [-2, 2]
    frequency_penalty: float = 0.0
    top_k: int = 0                   # sampling filters (host Sampler.set_filters): 0 = off; top_k in [0, 2^31 - 1]
    min_p: float = 0.0               # in [0, 1]
    seed: int = field(default_factory=lambda: int(time.time()))
    chat_template: Optional[str] = None
    max_seq_len: int = 0
    net_turbo: bool = True
    gpu_index: int = -1
    gpu_segments: Optional[str] = None
    benchmark: bool = False
    # GPU build extras
    gpus: int = 0            # spawn this many local ranks (0 = use the current torch.distributed world / single GPU)
    moe_mode: str = "auto"   # tp | ep | auto
    parallel: int = 1        # dllama-api: chat requests decoded together, one KV-cache slot each (1..8)
    parallel_cache: str = "split"   # dllama-api: the slots' KV-cache layout: split (floor(context / n) rows each) | paged (shared 64-row pages)
    kv_cache_float_type: str = "bf16"   # KV-cache storage: bf16 | q80 (int8 blocks of 32 with an f16 scale)
    draft_model: Optional[str] = None   # greedy speculative decoding: a smaller model with the same tokenizer drafts tokens
    draft_tokens: int = 3               # drafts per round: 1, 3 or 7 (checked by api.draft_refusal)


FLOAT_TYPES = ("f32", "f16", "q40", "q80")
KV_CACHE_FLOAT_TYPES = ("bf16", "q80")
MAX_TOP_K = 2**31 - 1
TEMPLATES = ("llama2", "llama3", "deepSeek3", "chatml")


def parse_args(argv: List[str], require_mode: bool) -> AppArgs:
    a = AppArgs()
    i = 0
    if require_mode and len(argv) > 0 and not argv[0].startswith("-"):
        a.mode = argv[0]
        i = 1
    if any(x in ("--usage", "--help", "-h") for x in argv):
        a.help = True
        return a
    while i < len(argv):
        name = argv[i]
        if i + 1 >= len(argv):
            raise ValueError(f"Missing value for option: {name}")
        value = argv[i + 1]
        if name == "--model":
            a.model = value
        elif name == "--tokenizer":
            a.tokenizer = value
        elif name == "--prompt":
            a.prompt = value
        elif name == "--buffer-float-type":
            if value not in FLOAT_TYPES:
                raise ValueError(f"Invalid float type: {value}")
            a.buffer_float_type = value
        elif name == "--workers":
            j = i + 1
            while j < len(argv) and not argv[j].startswith("-"):
                if ":" not in argv[j]:
                    raise ValueError(f"Invalid worker address: {argv[j]}")
                a.workers.append(argv[j])
                j += 1
            i = j
            continue
        elif name == "--port":
            a.port = int(value)
        elif name == "--host":
            a.host = value
        elif name == "--nthreads":
            a.nthreads = int(value)
            if a.nthreads < 1:
                raise ValueError("Number of threads must be at least 1")
        elif name == "--steps":
            a.steps = int(value)
        elif name == "--temperature":
            a.temperature = float(value)
        elif name == "--topp":
            a.topp = float(value)
        elif name in ("--presence-penalty", "--frequency-penalty"):
            v = float(value)
            if not -2.0 <= v <= 2.0:
                raise ValueError(f"{name} must be from -2 to 2")
            setattr(a, "presence_penalty" if name == "--presence-penalty" else "frequency_penalty", v)
        elif name == "--top-k":
            v = int(value)
            if not 0 <= v <= MAX_TOP_K:
                raise ValueError(f"--top-k must be an integer from 0 to {MAX_TOP_K}")
            a.top_k = v
        elif name == "--min-p":
            v = float(value)
            if not 0.0 <= v <= 1.0:
                raise ValueError("--min-p must be from 0 to 1")
            a.min_p = v
        elif name == "--seed":
            a.seed = int(value)
        elif name == "--chat-template":
            if value not in TEMPLATES:
                raise ValueError(f"Invalid chat template type: {value}")
            a.chat_template = value
        elif name == "--max-seq-len":
            a.max_seq_len = int(value)
        elif name == "--gpu-index":
            a.gpu_index = int(value)
        elif name == "--gpu-segments":
            if ":" not in value:
                raise ValueError("GPU segments expected in the format <from>:<to>")
            a.gpu_segments = value
        elif name == "--net-turbo":
            a.net_turbo = int(value) == 1
        elif name == "--gpus":
            a.gpus = int(value)
        elif name == "--moe-mode":
            a.moe_mode = value
        elif name == "--kv-cache-float-type":
            if value not in KV_CACHE_FLOAT_TYPES:
                raise ValueError(f"Invalid KV-cache float type: {value} (expected bf16 or q80)")
            a.kv_cache_float_type = value
        elif name == "--draft-model":
            a.draft_model = value
        elif name == "--draft-tokens":
            a.draft_tokens = int(value)
        elif name == "--parallel" and not require_mode:   # dllama-api only; its range is checked by api.parallel_refusal
            a.parallel = int(value)
        elif name == "--parallel-cache" and not require_mode:   # dllama-api only; checked by api.parallel_refusal
            a.parallel_cache = value
        else:
            raise ValueError(f"Unknown option: {name}")
        i += 2
    return a


USAGE = """Usage: dllama {inference|chat|perplexity|worker} {--model <path>} {--tokenizer <path>}
        [--prompt <text>] [--steps <n>] [--buffer-float-type {f32|f16|q40|q80}] [--max-seq-len <max>]
        [--temperature <temp>] [--topp <t>] [--presence-penalty <p>] [--frequency-penalty <f>] [--seed <s>]
        [--top-k <k>] [--min-p <p>]        sampling filters of sampled draws (default 0 = off)
        [--chat-template {llama2|llama3|deepSeek3|chatml}]
        [--kv-cache-float-type {bf16|q80}] KV-cache storage (default bf16; q80 = int8 blocks of 32 + f16 scale)
        [--draft-model <path>] [--draft-tokens {1|3|7}]
                                          greedy speculative decoding: the draft proposes k tokens (default 3) per round
        [--gpus <n>]                      run tensor-parallel on n local GPUs (spawns one process per GPU)
        [--workers <ip:port> ...] [--nthreads <n>] [--net-turbo {0|1}] [--gpu-index <i>] [--gpu-segments <a:b>]
                                          accepted for compatibility with the reference CLI
"""
