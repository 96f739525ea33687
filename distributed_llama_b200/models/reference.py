"""Pure-PyTorch f32 oracle of the three model families (correctness reference for the CUDA engine).

Implements the math of the graph the reference builds in src/llm.cpp:247-603 (embedding -> per layer
[rmsnorm, q/k/v, (qk-norm), rope, causal GQA attention, wo, residual] + [rmsnorm, SwiGLU FFN | MoE, residual]
-> final norm -> logits), on dequantised weights. `act_quant="q80"` additionally rounds activations to the
q80 grid wherever the reference casts to its q80 buffers (before every q40 matmul), so the CUDA kernels —
which do the same — can be compared tightly. `kv_quant="q80"` rounds every K/V row to the q80 grid as it is stored in the
cache (the engine's `--kv-cache-float-type q80`); every attention, the token's own row included, reads the rounded values.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from ..formats.model_file import ModelFile
from .config import ARCH_QWEN3, ARCH_QWEN3_MOE, ROPE_FALCON
from .. import host


def q80_round(x: torch.Tensor) -> torch.Tensor:
    """Round-trip through the q80 grid (per 32-element block: d = fp16(amax/127), q = round(x/d))."""
    shp = x.shape
    g = x.reshape(-1, 32).float()
    amax = g.abs().amax(dim=1, keepdim=True)
    d = amax / 127.0
    inv = torch.where(d != 0, 1.0 / d, torch.zeros_like(d))
    v = g * inv
    q = torch.sign(v) * torch.floor(v.abs() + 0.5)
    d16 = d.half().float()
    return (q * d16).reshape(shp)


class OracleModel:
    def __init__(self, model_file: ModelFile, act_quant: str = "none", device: str = "cpu", dtype=torch.float32,
                 kv_quant: str = "none"):
        if kv_quant not in ("none", "q80"):
            raise ValueError(f"unknown kv_quant {kv_quant!r}")
        self.mf = model_file
        self.h = h = model_file.header
        self.act_quant = act_quant
        self.kv_quant = kv_quant
        self.device = device
        self.dtype = dtype
        t = lambda name, l=0, e=0: torch.from_numpy(model_file.tensor_f32(model_file.entry(name, l, e))).to(device=device, dtype=dtype)
        self.embedding = t("embedding")
        self.layers = []
        for l in range(h.n_layers):
            L = {k: t("block_matmul_" + k, l) for k in ("q", "k", "v", "wo")}
            if h.n_experts > 0:
                L["gate"] = t("block_moe_gate", l)
                L["experts"] = [{k: t("block_matmul_" + k, l, e) for k in ("w1", "w2", "w3")} for e in range(h.n_experts)]
            else:
                for k in ("w1", "w2", "w3"):
                    L[k] = t("block_matmul_" + k, l)
            if h.qk_norm:
                L["q_norm"] = t("block_norm_q", l)
                L["k_norm"] = t("block_norm_k", l)
            L["norm_0"] = t("block_norm_0", l)
            L["norm_1"] = t("block_norm_1", l)
            self.layers.append(L)
        self.final_norm = t("final_norm")
        self.wcls = t("final_matmul_logits")
        rope = torch.from_numpy(np.asarray(host().build_rope_table(h, h.seq_len)))  # [seq, hd/2, 2]
        self.rope_cos = rope[..., 0].to(device=device, dtype=dtype)
        self.rope_sin = rope[..., 1].to(device=device, dtype=dtype)
        self.k_cache = [torch.zeros(h.seq_len, h.n_kv_heads, h.head_dim, device=device, dtype=dtype) for _ in range(h.n_layers)]
        self.v_cache = [torch.zeros(h.seq_len, h.n_kv_heads, h.head_dim, device=device, dtype=dtype) for _ in range(h.n_layers)]

    # -- pieces --
    def _aq(self, x):
        return q80_round(x).to(self.dtype) if self.act_quant == "q80" else x

    def _rms(self, x, w, eps):
        inv = torch.rsqrt(x.pow(2).mean(dim=-1, keepdim=True) + eps)
        return w * (x * inv)

    def _rope(self, x, pos):  # x [T, H, hd]
        cos = self.rope_cos[pos][:, None, :]
        sin = self.rope_sin[pos][:, None, :]
        if self.h.rope_type == ROPE_FALCON:
            half = x.shape[-1] // 2
            a, b = x[..., :half], x[..., half:]
            return torch.cat([a * cos - b * sin, a * sin + b * cos], dim=-1)
        a, b = x[..., 0::2], x[..., 1::2]
        out = torch.empty_like(x)
        out[..., 0::2] = a * cos - b * sin
        out[..., 1::2] = a * sin + b * cos
        return out

    def _ffn(self, y, w1, w2, w3):
        yq = self._aq(y)
        d = torch.nn.functional.silu(yq @ w1.T) * (yq @ w3.T)
        return self._aq(d) @ w2.T

    @torch.no_grad()
    def forward(self, tokens, start_pos: int) -> torch.Tensor:
        """tokens: sequence of T token ids occupying positions start_pos..start_pos+T-1. Returns logits [T, vocab]."""
        h = self.h
        tokens = torch.as_tensor(tokens, dtype=torch.long, device=self.device)
        T = tokens.numel()
        pos = torch.arange(start_pos, start_pos + T, device=self.device)
        x = self.embedding[tokens]
        eps = h.norm_epsilon
        kv_mul = h.n_heads // h.n_kv_heads
        for l, L in enumerate(self.layers):
            y = self._aq(self._rms(x, L["norm_0"], eps))
            q = (y @ L["q"].T).view(T, h.n_heads, h.head_dim)
            k = (y @ L["k"].T).view(T, h.n_kv_heads, h.head_dim)
            v = (y @ L["v"].T).view(T, h.n_kv_heads, h.head_dim)
            if h.qk_norm:
                q = self._rms(q, L["q_norm"], eps)
                k = self._rms(k, L["k_norm"], eps)
            q = self._rope(q, pos)
            k = self._rope(k, pos)
            if self.kv_quant == "q80":
                k, v = q80_round(k).to(self.dtype), q80_round(v).to(self.dtype)
            self.k_cache[l][start_pos:start_pos + T] = k
            self.v_cache[l][start_pos:start_pos + T] = v
            K = self.k_cache[l][: start_pos + T]
            V = self.v_cache[l][: start_pos + T]
            Kx = K.repeat_interleave(kv_mul, dim=1)   # [S, H, hd]
            Vx = V.repeat_interleave(kv_mul, dim=1)
            scores = torch.einsum("thd,shd->hts", q, Kx) / math.sqrt(h.head_dim)
            mask = torch.arange(start_pos + T, device=self.device)[None, :] > pos[:, None]
            scores = scores.masked_fill(mask[None], float("-inf"))
            att = torch.softmax(scores, dim=-1)
            z = torch.einsum("hts,shd->thd", att, Vx).reshape(T, h.q_dim)
            x = x + self._aq(z) @ L["wo"].T
            y = self._rms(x, L["norm_1"], eps)
            if h.n_experts > 0:
                probs = torch.softmax(y @ L["gate"].T, dim=-1)
                topv, topi = torch.topk(probs, h.n_active_experts, dim=-1)
                topv = topv / topv.sum(dim=-1, keepdim=True)
                out = torch.zeros_like(x)
                for t_i in range(T):
                    for j in range(h.n_active_experts):
                        E = L["experts"][int(topi[t_i, j])]
                        out[t_i] += topv[t_i, j] * self._ffn(y[t_i:t_i + 1], E["w1"], E["w2"], E["w3"])[0]
                x = x + out
            else:
                x = x + self._ffn(y, L["w1"], L["w2"], L["w3"])
        y = self._aq(self._rms(x, self.final_norm, eps))
        return y @ self.wcls.T

    def reset(self):
        for c in self.k_cache + self.v_cache:
            c.zero_()
