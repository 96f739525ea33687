"""Synthetic `.m` / `.t` generators (random-init weights in the real file layout).

There is no network access for checkpoints, so benchmarks and tests run on random weights written in
exactly the layout the converters produce (reference converter/convert-hf.py:59-104). Large models are
generated straight in the quantised domain (random nibbles + fp16 block scales chosen so activations stay
O(1)) which makes an 8B q40 file appear in seconds.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np

from ..formats import quants
from ..formats.model_file import write_model_header
from ..formats.tokenizer_file import write_tokenizer
from .config import ModelConfig, ARCH_QWEN3, ARCH_QWEN3_MOE

LLAMA3_TEMPLATE = (b"{% for message in messages %}{{'<|start_header_id|>' + message['role'] + '<|end_header_id|>\n\n'"
                   b" + message['content'] | trim + '<|eot_id|>'}}{% endfor %}"
                   b"{% if add_generation_prompt %}{{ '<|start_header_id|>assistant<|end_header_id|>\n\n' }}{% endif %}")
CHATML_TEMPLATE = (b"{% for message in messages %}{{'<|im_start|>' + message['role'] + '\n' + message['content'] + "
                   b"'<|im_end|>' + '\n'}}{% endfor %}{% if add_generation_prompt %}{{ '<|im_start|>assistant\n' }}{% endif %}")


class _TensorWriter:
    def __init__(self, f, seed: int):
        self.f = f
        self.rng = np.random.default_rng(seed)
        self.n_bytes = 0

    def _emit(self, raw: np.ndarray):
        self.f.write(memoryview(np.ascontiguousarray(raw)).cast("B"))
        self.n_bytes += raw.nbytes

    def matrix(self, float_type: int, d: int, n: int, std: Optional[float] = None, chunk_rows: int = 4096):
        std = std if std is not None else 1.0 / np.sqrt(n)
        if float_type == quants.F_Q40:
            # uniform nibbles -> value (nib-8)*delta has std ~4.61*delta
            delta = std / 4.61
            nb_row = n // 32
            for r0 in range(0, d, chunk_rows):
                rows = min(chunk_rows, d - r0)
                blk = np.empty((rows * nb_row, 18), dtype=np.uint8)
                scales = (delta * self.rng.uniform(0.7, 1.3, size=rows * nb_row)).astype(np.float16)
                blk[:, 0:2] = scales.view(np.uint8).reshape(-1, 2)
                blk[:, 2:] = np.frombuffer(self.rng.bytes(rows * nb_row * 16), dtype=np.uint8).reshape(-1, 16)
                self._emit(blk)
        else:
            for r0 in range(0, d, chunk_rows):
                rows = min(chunk_rows, d - r0)
                x = self.rng.standard_normal((rows, n), dtype=np.float32) * np.float32(std)
                self._emit(quants.quantize(float_type, x))

    def norm(self, n: int, gain: float = 1.0):
        x = (1.0 + 0.1 * self.rng.standard_normal(n, dtype=np.float32)).astype(np.float32) * np.float32(gain)
        self._emit(x)


def write_synthetic_model(path: str, cfg: ModelConfig, weights_float_type: int = quants.F_Q40, seed: int = 1234,
                          attn_gain: float = 1.0) -> int:
    """Writes a random-weight model file for `cfg`; returns the file size in bytes.

    `attn_gain` scales the attention scores: it multiplies the std of the q and k matrices, or, for models with QK-norm
    (where the norm weights set the score scale), the q/k norm weights. It draws no extra random numbers: every other
    tensor is the same for any gain, and the default of 1.0 leaves the whole file unchanged."""
    tmp = path + ".tmp"
    head_dim = cfg.head_dim or cfg.dim // cfg.n_heads
    q_dim, kv_dim = head_dim * cfg.n_heads, head_dim * cfg.n_kv_heads
    ff = cfg.moe_hidden_dim if cfg.arch_type == ARCH_QWEN3_MOE else cfg.hidden_dim
    wt = weights_float_type
    qk_norm = cfg.arch_type in (ARCH_QWEN3, ARCH_QWEN3_MOE)
    qk_std = (1.0 if qk_norm else attn_gain) / np.sqrt(cfg.dim)
    with open(tmp, "wb") as f:
        write_model_header(f, cfg.header_params(wt))
        w = _TensorWriter(f, seed)
        w.matrix(quants.F_32, cfg.vocab_size, cfg.dim, std=1.0)
        for _ in range(cfg.n_layers):
            w.matrix(wt, q_dim, cfg.dim, std=qk_std)
            w.matrix(wt, kv_dim, cfg.dim, std=qk_std)
            w.matrix(wt, kv_dim, cfg.dim)
            w.matrix(wt, cfg.dim, q_dim, std=0.5 / np.sqrt(q_dim))
            if cfg.n_experts > 0:
                w.matrix(quants.F_32, cfg.n_experts, cfg.dim, std=1.0 / np.sqrt(cfg.dim))
                for _e in range(cfg.n_experts):
                    w.matrix(wt, ff, cfg.dim)
                    w.matrix(wt, cfg.dim, ff, std=0.5 / np.sqrt(ff))
                    w.matrix(wt, ff, cfg.dim)
            else:
                w.matrix(wt, ff, cfg.dim)
                w.matrix(wt, cfg.dim, ff, std=0.5 / np.sqrt(ff))
                w.matrix(wt, ff, cfg.dim)
            if qk_norm:
                w.norm(head_dim, attn_gain)
                w.norm(head_dim, attn_gain)
            w.norm(cfg.dim)
            w.norm(cfg.dim)
        w.norm(cfg.dim)
        w.matrix(wt, cfg.vocab_size, cfg.dim)
    os.replace(tmp, path)
    return os.path.getsize(path)


def write_synthetic_tokenizer(path: str, vocab_size: int, style: str = "llama3") -> None:
    """A byte-level BPE-shaped vocabulary: 256 byte tokens, a few hundred real merges, filler tokens up to
    bosId, then special tokens. Respects the reference's `regularVocabSize == bosId` assumption
    (reference src/tokenizer.cpp:138-140) so the reference binary can load it too."""
    if style == "llama3":
        specials = [b"<|begin_of_text|>", b"<|end_of_text|>", b"<|start_header_id|>", b"<|end_header_id|>", b"<|eot_id|>"]
        bos_name, eos_names, template = b"<|begin_of_text|>", [b"<|end_of_text|>", b"<|eot_id|>"], LLAMA3_TEMPLATE
    elif style == "chatml":
        specials = [b"<|endoftext|>", b"<|im_start|>", b"<|im_end|>"]
        bos_name, eos_names, template = b"<|endoftext|>", [b"<|im_end|>", b"<|endoftext|>"], CHATML_TEMPLATE
    else:
        raise ValueError(style)
    n_special = max(len(specials), 16 if vocab_size >= 1024 else len(specials))
    while len(specials) < n_special:
        specials.append(b"<|reserved_special_token_%d|>" % len(specials))
    n_regular = vocab_size - len(specials)
    if n_regular < 256:
        raise ValueError("vocab too small")
    tokens = [bytes([b]) if b else b"\x00" for b in range(256)]
    seen = set(tokens)
    words = [b" the", b" and", b" of", b" to", b" in", b" is", b" that", b" it", b" for", b" with", b" was", b" on",
             b"Hello", b" world", b" model", b" token", b" llama", b" hello", b" you", b" are", b"ing", b"er", b"ed",
             b"tion", b" a", b" I", b"\n\n", b"user", b"assistant", b"system", b" What", b" how", b"?", b"!"]
    # every prefix chain needed so that pair merges can actually build the word
    for wd in words:
        for k in range(2, len(wd) + 1):
            piece = wd[:k]
            if piece not in seen and len(tokens) < n_regular:
                tokens.append(piece)
                seen.add(piece)
    i = 0
    while len(tokens) < n_regular:
        piece = b"\xc4\xa0tok%d" % i   # 'Ġtok<i>' — never produced by ASCII text segmentation
        i += 1
        if piece not in seen:
            tokens.append(piece)
            seen.add(piece)
    bos_id = len(tokens)
    tokens += specials
    scores = [-float(j) for j in range(len(tokens))]
    eos_ids = [tokens.index(e) for e in eos_names]
    assert tokens[bos_id] == bos_name
    write_tokenizer(path, tokens, scores, template, bos_id, True, eos_ids)
