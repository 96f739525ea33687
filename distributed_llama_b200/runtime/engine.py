"""Python handle of the native per-rank engine (csrc/cuda/engine.cu).

Owns the device tensors (weights, KV cache, the activation buffers it reads), hands their pointers to the C++ engine and exposes
the three calls the apps need: `prefill(tokens, pos)`, `step(token, pos)` -> logits, and the device-resident greedy
decode loop `decode_greedy(n)` that replays the captured CUDA graph.
Plays the role of the reference's RootLlmInference (src/app.cpp:168-208): setBatchSize/setPosition/setToken/forward.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from ..models.loader import DeviceWeights
from ..ops import cuda_lib as cl


def _p(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def logprobs_rows(logits: torch.Tensor, chosen: torch.Tensor, k: Sequence[int], row_mask: Optional[int] = None,
                  bias: Optional[torch.Tensor] = None, counts: Optional[torch.Tensor] = None, presence: float = 0.0,
                  frequency: float = 0.0, row_params: Optional[torch.Tensor] = None, shared_row: bool = False) -> torch.Tensor:
    """The log-probability kernel (csrc/cuda/logprobs.cu) on explicit device buffers: B = len(k) rows of `logits` ([B][n] f32,
    or one row read by every row with shared_row), chosen ([B] int32: each row's draw; counts are those after it), k[b] top
    entries, rows outside row_mask (default: all) untouched. Optional controls: bias ([n], or [B][n]: one per row) f32, counts
    [B][n] int32, and the penalties, per row through row_params ([B][4] f32, columns 2 and 3). Returns the device result blocks
    [B][LOGPROBS_WORDS] int32 (ops.cuda_lib.decode_logprobs reads one)."""
    B = len(k)
    n = logits.shape[-1]
    mask = ((1 << B) - 1) if row_mask is None else int(row_mask)
    out = torch.zeros(B, cl.LOGPROBS_WORDS, dtype=torch.int32, device=logits.device)
    ks = (C.c_int32 * B)(*[int(x) for x in k])
    stride = 0 if shared_row or logits.dim() == 1 else logits.stride(0)
    bias_stride = bias.stride(0) if bias is not None and bias.dim() == 2 else 0
    counts_stride = counts.stride(0) if counts is not None and counts.dim() == 2 else 0
    cl.check(cl.lib().dl_logprobs_rows(logits.data_ptr(), stride, n, B, mask, ks, chosen.data_ptr(), _p(bias), bias_stride, _p(counts),
                                       counts_stride, float(presence), float(frequency), _p(row_params), out.data_ptr(), cl.stream_ptr()),
             "logprobs_rows")
    return out


def _plan_chunks(call) -> List[tuple]:
    cap = 64
    while True:
        out = (C.c_uint32 * (3 * cap))()
        n = call(out, cap)
        cl.check(min(n, 0), "prefill_plan")
        if n <= cap:
            return [(int(out[3 * i]), int(out[3 * i + 1]), bool(out[3 * i + 2])) for i in range(n)]
        cap = n


def prefill_plan(n: int, start_pos: int, rows: int, max_prefill: int, max_batch: int, min_tc: int, tensor_cores: bool,
                 slot: int = -1, slots: int = 1) -> List[tuple]:
    """The chunks the engine splits a prompt of n tokens at start_pos into (dl_prefill_plan; no device needed), in a cache of `rows`
    rows: (T, first position, on the tensor cores) per chunk. Raises on a prompt past the cache (code -60) or a slot prefill
    without slots (-64)."""
    return _plan_chunks(lambda out, cap: cl.lib().dl_prefill_plan(n, start_pos, slot, slots, rows, max_prefill, max_batch, min_tc,
                                                                  1 if tensor_cores else 0, out, cap))


def dense_max_batch(max_batch: int, dim: int, ff_dim: int, q_dim: int) -> int:
    """Largest power-of-two batch <= max_batch that the dense-weight GEMV holds: it stages the f32 activations of all tokens of a
    launch in shared memory (gemv_dense.cu), so the widest matrix row (dim, ff_dim or q_dim values) bounds it."""
    widest = max(dim, ff_dim, q_dim)
    cap = (200 * 1024) // (4 * widest)
    if cap < 1:
        raise ValueError("matrix rows too wide for the dense-weight kernels on one GPU; use more ranks")
    while max_batch > cap:
        max_batch //= 2
    return max_batch


class Engine:
    def __init__(self, weights: DeviceWeights, max_batch: int = 8, n_splits: int = 0, use_pdl: bool = True,
                 seq_len: Optional[int] = None, comm=None, max_prefill: int = 192, collectives: str = "auto",
                 kv_cache_float_type: str = "bf16"):
        if kv_cache_float_type not in cl.KV_CACHE_TYPES:
            raise ValueError(f"unknown KV-cache float type {kv_cache_float_type!r} (expected one of: {', '.join(cl.KV_CACHE_TYPES)})")
        self.kv_cache_float_type = kv_cache_float_type
        self.w = w = weights
        h = w.header
        dev = w.embedding.device
        self.device = dev
        self.seq_len = seq_len or h.seq_len
        if h.n_experts > 0:
            max_batch = 1          # the MoE kernels route one token per launch
        self.dense = getattr(w, "weight_kind", 0) != 0
        if self.dense:
            max_batch = dense_max_batch(max_batch, h.dim, w.ff_dim, w.n_heads * h.head_dim)
        self.max_batch = max_batch
        self.max_prefill = min(max_prefill, 256)
        props = torch.cuda.get_device_properties(dev)
        self.num_sms = props.multi_processor_count
        if n_splits <= 0:
            n_splits = max(1, min(32, (2 * self.num_sms) // max(1, w.n_heads)))
        self.n_splits = n_splits
        hd = h.head_dim
        q_dim, kv_dim = w.n_heads * hd, w.n_kv_heads * hd
        self.qkv_dim = q_dim + 2 * kv_dim
        f32 = dict(dtype=torch.float32, device=dev)
        self.tokens = torch.zeros(max_batch, dtype=torch.int32, device=dev)
        self.pos = torch.zeros(max_batch, dtype=torch.int32, device=dev)
        self.x = torch.zeros(max_batch, h.dim, **f32)
        self.logits = torch.zeros(max_batch, w.vocab, **f32)
        self.history = torch.zeros(self.seq_len + 1, dtype=torch.int32, device=dev)
        if kv_cache_float_type == "q80":
            # int8 values [nKvHeads][seqLen][hd] and f16 scales [nKvHeads][seqLen][hd / 32] (+ 8 halves of tail padding: the
            # persistent kernel copies the 16-byte aligned span around a chunk's scale rows)
            kv_shape, kv_dtype = (w.n_kv_heads, self.seq_len, hd), torch.int8
            sc_elems = w.n_kv_heads * self.seq_len * (hd // 32)
            self.k_scale = [torch.zeros(sc_elems + 8, dtype=torch.float16, device=dev) for _ in range(h.n_layers)]
            self.v_scale = [torch.zeros(sc_elems + 8, dtype=torch.float16, device=dev) for _ in range(h.n_layers)]
        else:
            kv_shape, kv_dtype = (w.n_kv_heads, self.seq_len, hd), torch.bfloat16
            self.k_scale = self.v_scale = [None] * h.n_layers
        self.k_cache = [torch.zeros(*kv_shape, dtype=kv_dtype, device=dev) for _ in range(h.n_layers)]
        self.v_cache = [torch.zeros(*kv_shape, dtype=kv_dtype, device=dev) for _ in range(h.n_layers)]

        cfg = cl.EngineConfig(dim=h.dim, nLayers=h.n_layers, nHeads=w.n_heads, nKvHeads=w.n_kv_heads, headDim=hd,
                              ffDim=w.ff_dim, vocab=w.vocab, seqLen=self.seq_len, nExperts=h.n_experts,
                              nActiveExperts=h.n_active_experts, maxBatch=max_batch, nSplits=n_splits, rank=w.rank,
                              nRanks=w.n_ranks, numSms=self.num_sms, eps=h.norm_epsilon, usePdl=1 if use_pdl else 0,
                              moeFirstExpert=w.first_expert, moeNumLocal=w.n_local_experts,
                              wType=getattr(w, "weight_kind", 0),
                              hiddenAct=1 if int(h.hidden_act) == 0 else 0,   # header: ACT_GELU = 0, ACT_SILU = 1
                              kvType=cl.KV_CACHE_TYPES[kv_cache_float_type], maxPrefill=self.max_prefill)
        self._lib = cl.lib()
        self._h = self._lib.dl_engine_create(C.byref(cfg))
        if not self._h:
            raise RuntimeError("dl_engine_create failed: unsupported configuration or out of device memory")
        for l, L in enumerate(w.layers):
            lp = cl.LayerPtrs(qkvQs=_p(L.qkv.qs), qkvSc=_p(L.qkv.scales), woQs=_p(L.wo.qs), woSc=_p(L.wo.scales),
                              w13Qs=_p(L.w13.qs), w13Sc=_p(L.w13.scales), w2Qs=_p(L.w2.qs), w2Sc=_p(L.w2.scales),
                              norm0=_p(L.norm0), norm1=_p(L.norm1), qNorm=_p(L.q_norm), kNorm=_p(L.k_norm),
                              moeGate=_p(L.moe_gate), kCache=_p(self.k_cache[l]), vCache=_p(self.v_cache[l]),
                              kScale=_p(self.k_scale[l]), vScale=_p(self.v_scale[l]))
            cl.check(self._lib.dl_engine_set_layer(self._h, l, C.byref(lp)), "engine_set_layer")
        emb_peers = (C.c_void_p * 8)(*([C.c_void_p(p) for p in (w.embedding_ptrs or [])] + [None] * (8 - len(w.embedding_ptrs or []))))
        gp = cl.GlobalPtrs(embedding=_p(w.embedding), embeddingPeers=emb_peers, embRowsPerRank=w.embedding_rows or 0, finalNorm=_p(w.final_norm), wclsQs=_p(w.wcls.qs),
                           wclsSc=_p(w.wcls.scales), rope=_p(w.rope), vocabFull=h.vocab_size, tokens=_p(self.tokens),
                           pos=_p(self.pos), x=_p(self.x), logits=_p(self.logits), history=_p(self.history))
        cl.check(self._lib.dl_engine_set_globals(self._h, C.byref(gp)), "engine_set_globals")
        self.comm = comm
        tp = comm is not None and comm.world_size > 1
        # Collectives: "fused" = inside the kernels over NVLink peer memory (ranks of one node, q40 weights);
        # "nccl" = library all-reduce between kernel groups (ranks on several nodes, dense weight files, DL_COLLECTIVES=nccl).
        self.collectives = "fused"
        if tp and (collectives == "nccl" or os.environ.get("DL_COLLECTIVES") == "nccl" or self.dense
                   or not getattr(comm, "single_node", True)):
            self.collectives = "nccl"
        if tp and self.collectives == "fused":
            comm.alloc_arena(self._lib.dl_engine_arena_bytes(self._h))
            cp = comm.comm_ptrs()
            cl.check(self._lib.dl_engine_set_comm(self._h, C.byref(cp)), "engine_set_comm")
        self._parts = tp and self.collectives == "nccl"
        self._ybuf = torch.zeros(max_batch, h.dim, **f32)
        self._tc_min = 9
        self.mega = False
        if h.n_experts == 0 and not self.dense and not self._parts and os.environ.get("DL_NO_MEGA") is None:
            self.enable_mega(True)     # persistent decode kernel by default; the engine falls back per call if a shape is unsupported
        self.slots, self.slot_len, self.paged = 1, self.seq_len, False
        self._stage_tok = torch.zeros(max_batch, dtype=torch.int32).pin_memory()
        self._stage_pos = torch.zeros(max_batch, dtype=torch.int32).pin_memory()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.dl_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def set_vocab_limit(self, limit: int):
        """Greedy arg-max on the device never returns ids >= limit (the tokenizer's vocabulary size: embeddings may be padded
        beyond it, reference src/app.cpp:243-246 builds its sampler on the tokenizer size too)."""
        cl.check(self._lib.dl_engine_set_vocab_limit(self._h, int(limit)), "engine_set_vocab_limit")

    # -- device-side sampling --
    def seed_sampler(self, seed: int):
        """Seeds the device-resident generator (same xorshift* stream as the host Sampler). Every rank must use the same seed."""
        cl.check(self._lib.dl_engine_sampler_seed(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF), "engine_sampler_seed")
        self._sampler_ready = True

    def step_sampled(self, token: int, pos: int, temperature: float, topp: float) -> None:
        """Forward of one token + temperature/top-p sampling on the device (csrc/cuda/sampler.cu); the sampled token lands in
        tokens[0] and history[pos + 1]. No logits leave the GPU; under tensor parallelism the vocabulary slices are exchanged
        through peer memory and every rank draws the same token."""
        if not getattr(self, "_sampler_ready", False):
            raise RuntimeError("seed_sampler() must be called first")
        self.forward_batch([token], pos, logits_mode=1)
        cl.check(self._lib.dl_engine_sample(self._h, float(temperature), float(topp), cl.stream_ptr()), "engine_sample")

    def set_sampling_controls(self, presence: float, frequency: float, bias: Sequence, row_mask: int) -> None:
        """Presence / frequency penalties and logit bias ((id, value) pairs) of the following device draws; zeroes the count
        rows in row_mask (bit 0: single sequence, bit 1 + i: choice i). All zero and no bias: off. Every rank makes the same
        call. With controls on, step_sampled and the choices steps accept temperature 0 (arg-max of the controlled logits)."""
        n = len(bias)
        ids = (C.c_int32 * max(n, 1))(*[int(t) for t, _ in bias])
        vals = (C.c_float * max(n, 1))(*[float(v) for _, v in bias])
        cl.check(self._lib.dl_engine_set_sampling_controls(self._h, float(presence), float(frequency), ids, vals, n, int(row_mask),
                                                            cl.stream_ptr()),
                 "engine_set_sampling_controls")
        if presence or frequency or n:
            self._sampler_ready = True

    def set_sampling_filters(self, top_k: int, min_p: float) -> None:
        """top_k / min_p of the following sampled device draws of the single sequence and the choices (host Sampler.set_filters
        defines them); 0 / 0.0: off. They persist until changed; temperature-0 draws ignore them. Every rank makes the same call."""
        cl.check(self._lib.dl_engine_set_sampling_filters(self._h, int(top_k), float(min_p)), "engine_set_sampling_filters")

    # -- choices: several completions of one prompt, one row per choice (csrc/cuda/attn_decode.cu) --
    def supports_choices(self, n: int) -> bool:
        """True if n choices can run as one batched step: dense layers, kernel-fused collectives, n <= max_batch."""
        return 1 <= n <= min(8, self.max_batch) and self.w.header.n_experts == 0 and not self._parts

    @staticmethod
    def _choice_batch(n: int, active: Optional[Sequence[bool]] = None):
        """(rows padded to a power of two, bit mask of the inactive rows: finished choices and padding)."""
        nb = 1
        while nb < n:
            nb *= 2
        mask = 0
        for b in range(nb):
            if b >= n or (active is not None and not active[b]):
                mask |= 1 << b
        return nb, mask

    def seed_choice_samplers(self, seeds: Sequence[int]):
        """Seeds generator i of the batched sampler with seeds[i]; the single-sequence generator keeps its stream."""
        arr = (C.c_uint64 * len(seeds))(*[int(s) & 0xFFFFFFFFFFFFFFFF for s in seeds])
        cl.check(self._lib.dl_engine_sampler_seed_rows(self._h, arr, len(seeds)), "engine_sampler_seed_rows")
        self._sampler_ready = True

    def sample_choices_first(self, n: int, temperature: float, topp: float) -> None:
        """After a single-token forward at the prompt end: choice i draws its first token from that logits row with generator i.
        The draws land in tokens[:n]."""
        nb, mask = self._choice_batch(n)
        cl.check(self._lib.dl_engine_sample_rows(self._h, nb, mask, float(temperature), float(topp), 1, cl.stream_ptr()), "engine_sample_rows")

    def choices_forward(self, tokens: Sequence[int], P: int, C: int, j: int, active: Optional[Sequence[bool]] = None) -> None:
        """One choices step: choice b feeds tokens[b] at rotary position P + 1 + j, attends to the prompt rows [0, P] and its own
        rows [P + 1 + b*C, P + 1 + b*C + j], and stores its K/V at the last of those. Inactive choices write nothing.
        Logits of every row land in logits[:len(tokens)]."""
        n = len(tokens)
        nb, mask = self._choice_batch(n, active)
        if not self.supports_choices(n):
            raise ValueError("batched choices need dense layers, kernel-fused collectives and n <= max_batch")
        if C < 1 or j >= C or P + 1 + n * C > self.seq_len:
            raise ValueError("choice rows beyond the context length")
        self.tokens[:nb].copy_(torch.tensor(list(tokens) + [0] * (nb - n), dtype=torch.int32))
        self.pos[:nb].fill_(P + 1 + j)
        cl.check(self._lib.dl_engine_choices_forward(self._h, nb, P, C, j, mask, cl.stream_ptr()), "engine_choices_forward")

    def choices_first(self, token: int, P: int, n: int, temperature: float, topp: float, logprobs: Optional[int] = None) -> List[int]:
        """Forward of the prompt's last token at P, then choice i draws its first token from that row with generator i.
        logprobs = k: also the log-probabilities of every draw (read_logprobs())."""
        self.forward_batch([token], P, logits_mode=1)
        self.sample_choices_first(n, temperature, topp)
        if logprobs is not None:
            self.logprobs([logprobs] * n, (1 << n) - 1, first_row=1, controlled=True, shared_row=True)
        out = self.tokens[:n].tolist()
        self.check_abort()
        return out

    def choices_step(self, tokens: Sequence[int], P: int, C: int, j: int, active: Sequence[bool], temperature: float,
                     topp: float, logprobs: Optional[int] = None) -> List[int]:
        """choices_forward, then every active row draws its next token with its own generator. Returns the draws (inactive
        rows: whatever tokens[] held). logprobs = k: also the log-probabilities of the active rows' draws (read_logprobs())."""
        self.choices_forward(tokens, P, C, j, active)
        nb, mask = self._choice_batch(len(tokens), active)
        cl.check(self._lib.dl_engine_sample_rows(self._h, nb, mask, float(temperature), float(topp), 0, cl.stream_ptr()), "engine_sample_rows")
        if logprobs is not None:
            self.logprobs([logprobs] * len(tokens), sum(1 << b for b in range(len(tokens)) if active[b]), first_row=1, controlled=True)
        out = self.tokens[:len(tokens)].tolist()
        self.check_abort()
        return out

    # -- KV-cache slots: up to 8 independent sequences decoded together (csrc/cuda/attn_decode.cu) --
    def set_slots(self, n: int, layout: str = "split") -> None:
        """Splits every layer's KV cache into n slots of floor(seq_len / n) rows (layout "split"), or lets n slots share it as
        one pool of 64-row pages (layout "paged": slot_len is 64 * floor(seq_len / 64), and a slot's rows must be reserved with
        slot_reserve before a step or prefill writes them). Single GPU, dense q40 layers only; n = 1 is the ordinary
        single-sequence engine."""
        if layout not in cl.SLOT_CACHE_LAYOUTS:
            raise ValueError(f"unknown KV-cache slot layout {layout!r} (expected split or paged)")
        if self.slots > 1:   # the layout is chosen while the cache is not split
            cl.check(self._lib.dl_engine_set_slots(self._h, 1), "engine_set_slots")
        cl.check(self._lib.dl_engine_set_slot_cache(self._h, 1 if layout == "paged" else 0), "engine_set_slot_cache")
        cl.check(self._lib.dl_engine_set_slots(self._h, int(n)), "engine_set_slots")
        self.slots = int(n)
        self.paged = layout == "paged" and n > 1
        self.slot_len = int(self._lib.dl_engine_slot_len(self._h))

    def slot_reserve(self, slot: int, rows: int) -> bool:
        """Paged slots: grows slot `slot`'s pages to cover rows [0, rows), lowest free pages first. False, with nothing changed,
        when the pool has too few free pages."""
        rc = self._lib.dl_engine_slot_reserve(self._h, int(slot), int(rows))
        if rc == cl.POOL_SHORT:
            return False
        cl.check(rc, "engine_slot_reserve")
        return True

    def slot_trim(self, slot: int, rows: int) -> None:
        """Paged slots: keeps the pages of rows [0, rows) of slot `slot` and returns the rest to the pool."""
        cl.check(self._lib.dl_engine_slot_trim(self._h, int(slot), int(rows)), "engine_slot_trim")

    def slot_release(self, slot: int) -> None:
        """Paged slots: returns slot `slot`'s pages to the pool."""
        cl.check(self._lib.dl_engine_slot_release(self._h, int(slot)), "engine_slot_release")

    def free_pages(self) -> int:
        return int(self._lib.dl_engine_free_pages(self._h))

    def slot_pages(self, slot: int) -> List[int]:
        """Paged slots: slot `slot`'s physical pages in logical order."""
        cap = max(1, self.seq_len // cl.PAGE_ROWS)
        out = (C.c_int32 * cap)()
        n = self._lib.dl_engine_slot_pages(self._h, int(slot), out, cap)
        if n < 0:
            cl.check(n, "engine_slot_pages")
        return list(out[:n])

    def slot_prefill(self, slot: int, tokens: Sequence[int], start_pos: int) -> None:
        """Feeds tokens at positions start_pos.. into slot `slot` (tensor-core prefill kernels with the slot's cache). No logits."""
        tokens = list(tokens)
        if start_pos + len(tokens) > self.slot_len:
            raise ValueError("position beyond the slot length")
        self._prefill(tokens, start_pos, int(slot), False)

    def slot_copy(self, src: int, dst: int, P: int) -> None:
        """Copies rows [0, P) of slot src into slot dst (every layer and KV head); paged slots: into dst's own pages, reserved
        first (RuntimeError with code -68 when the pool is short)."""
        cl.check(self._lib.dl_engine_slot_copy(self._h, int(src), int(dst), int(P), cl.stream_ptr()), "engine_slot_copy")

    def slot_sampling(self, slot: int, seed: int, temperature: float, topp: float, presence: float = 0.0, frequency: float = 0.0,
                      bias: Sequence = (), *, top_k: int = 0, min_p: float = 0.0) -> None:
        """Seeds slot `slot`'s generator, zeroes its token counts and sets its temperature (0: arg-max), top-p, penalties,
        logit bias ((id, value) pairs) and sampling filters (top_k / min_p, 0: off)."""
        n = len(bias)
        ids = (C.c_int32 * max(n, 1))(*[int(t) for t, _ in bias])
        vals = (C.c_float * max(n, 1))(*[float(v) for _, v in bias])
        cl.check(self._lib.dl_engine_slot_sampling(self._h, int(slot), int(seed) & 0xFFFFFFFFFFFFFFFF, float(temperature), float(topp),
                                                    float(presence), float(frequency), ids, vals, n, cl.stream_ptr()),
                 "engine_slot_sampling")
        if top_k or min_p:
            cl.check(self._lib.dl_engine_slot_filters(self._h, int(slot), int(top_k), float(min_p)), "engine_slot_filters")

    def _slot_args(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]):
        n = self.slots
        mask = sum(1 << b for b in range(n) if not active[b])
        return (C.c_int32 * n)(*[int(t) for t in tokens]), (C.c_int32 * n)(*[int(p) for p in pos]), mask

    def slots_forward(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]) -> torch.Tensor:
        """Row b feeds tokens[b] at position pos[b] of slot b (active rows only). Returns the logits rows [slots][vocab]."""
        t, p, mask = self._slot_args(tokens, pos, active)
        cl.check(self._lib.dl_engine_slots_forward(self._h, t, p, mask, cl.stream_ptr()), "engine_slots_forward")
        return self.logits[:self.slots]

    def slots_step(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]) -> List[int]:
        """slots_forward, then every active row draws its next token with its slot's settings. Returns the draws (inactive
        rows: -1)."""
        t, p, mask = self._slot_args(tokens, pos, active)
        out = (C.c_int32 * self.slots)(*([-1] * self.slots))
        cl.check(self._lib.dl_engine_slots_step(self._h, t, p, mask, out, cl.stream_ptr()), "engine_slots_step")
        self.check_abort()
        return list(out)

    def slot_logprobs(self, slot: int, k: Optional[int]) -> None:
        """Log-probabilities of slot `slot`'s draws with k top entries (None: off, as after every slot_sampling)."""
        cl.check(self._lib.dl_engine_slot_logprobs(self._h, int(slot), -1 if k is None else int(k)), "engine_slot_logprobs")

    def slots_step_logprobs(self, tokens: Sequence[int], pos: Sequence[int], active: Sequence[bool]):
        """slots_step that also returns, per slot, the log-probabilities of its draw (see logprobs) for the active slots whose
        logprobs are on (slot_logprobs), None for the others."""
        t, p, mask = self._slot_args(tokens, pos, active)
        out = (C.c_int32 * self.slots)(*([-1] * self.slots))
        lp = (C.c_int32 * (self.slots * cl.LOGPROBS_WORDS))()
        for b in range(self.slots):
            lp[b * cl.LOGPROBS_WORDS + 2] = -1   # rows the step leaves alone keep k = -1
        cl.check(self._lib.dl_engine_slots_step_logprobs(self._h, t, p, mask, out, lp, cl.stream_ptr()), "engine_slots_step_logprobs")
        self.check_abort()
        W = cl.LOGPROBS_WORDS
        rows = [None if lp[b * W + 2] < 0 else cl.decode_logprobs(lp[b * W:(b + 1) * W]) for b in range(self.slots)]
        return list(out), rows

    # -- per-token log-probabilities of the last draw (csrc/cuda/logprobs.cu) --
    def logprobs(self, k: Sequence[int], row_mask: int = 1, first_row: int = 0, controlled: bool = False, shared_row: bool = False) -> None:
        """Enqueues, behind the last draw on the current stream, the log-probabilities of the tokens in tokens[b] for the rows b set
        in row_mask: logprob(i) = x[i] - logsumexp(x) over the sampled vocabulary of logits row b (row 0 for every row with
        shared_row), x the logits after the sampling controls the draw used when `controlled` (count row first_row + b), and the
        k[b] largest entries. The result block is copied to pinned memory on the same stream: read it with read_logprobs() after
        the stream has been synchronised (the token copy that follows does that)."""
        rows = len(k)
        if not hasattr(self, "lp_out"):
            self.lp_out = torch.zeros(self.max_batch, cl.LOGPROBS_WORDS, dtype=torch.int32, device=self.device)
            self._lp_host = torch.zeros(self.max_batch, cl.LOGPROBS_WORDS, dtype=torch.int32).pin_memory()
        ks = (C.c_int32 * rows)(*[int(x) for x in k])
        flags = (cl.LP_CONTROLLED if controlled else 0) | (cl.LP_SHARED_ROW if shared_row else 0)
        cl.check(self._lib.dl_engine_logprobs(self._h, rows, int(row_mask), ks, int(first_row), flags, self.lp_out.data_ptr(), cl.stream_ptr()),
                 "engine_logprobs")
        self._lp_host[:rows].copy_(self.lp_out[:rows], non_blocking=True)
        self._lp_mask, self._lp_rows = int(row_mask), rows

    def read_logprobs(self) -> list:
        """The rows of the last logprobs() call, once its stream is synchronised: (chosen id, logprob, [(id, logprob), ...]) per row
        of its mask, None for the other rows."""
        h = self._lp_host.numpy()
        return [cl.decode_logprobs(h[b]) if (self._lp_mask >> b) & 1 else None for b in range(self._lp_rows)]

    def logprobs_host_draw(self, chosen: int, k: int, sampler) -> tuple:
        """Log-probabilities of a token the host sampler drew from logits[0] of the last forward (single GPU): the same kernel on
        the device logits, with the sampler's controls and its counts after the draw uploaded. Returns the decoded row."""
        dev = self.device
        bias = counts = None
        if sampler.controls_active:
            n = sampler.vocab_size
            bias = torch.zeros(n, dtype=torch.float32)
            for t, v in sampler.logit_bias:
                bias[t] = v
            bias = bias.to(dev)
            counts = torch.as_tensor(np.asarray(sampler.counts, dtype=np.uint32).view(np.int32)).reshape(1, -1).to(dev)
        n = min(sampler.vocab_size, self.w.vocab)
        out = logprobs_rows(self.logits[0:1, :n], torch.tensor([chosen], dtype=torch.int32, device=dev), [k], bias=bias, counts=counts,
                            presence=sampler.presence_penalty, frequency=sampler.frequency_penalty)
        return cl.decode_logprobs(out[0].cpu().tolist())

    def sampler_state(self) -> int:
        """State of the single-sequence device generator (0 before the first seeding); seed_sampler(state) continues its stream."""
        return int(self._lib.dl_engine_sampler_state(self._h))

    # -- traffic / synchronisation accounting (reference: NnNetwork::getStats + executor sync timers, src/dllama.cpp:59-66) --
    def sync_ns(self) -> int:
        """Cumulative ns the decode kernel waited for peer ranks inside its fused all-reduces (0 on one GPU)."""
        return int(self._lib.dl_engine_sync_ns(self._h))

    def link_bytes(self, n_tokens: int) -> tuple:
        """(sent, received) NVLink bytes of this rank for a forward over n_tokens tokens: 2 all-reduces per layer, every value
        travels as an 8-byte LL word; with the NVSwitch multicast mapping a value is sent once and replicated by the switch."""
        n = self.comm.world_size if (self.comm is not None and not self._parts) else 1
        if n <= 1:
            return 0, 0
        h = self.w.header
        per_ar = n_tokens * h.dim * 8
        mc = 1 if getattr(self.comm, "mc_ptr", 0) and n_tokens == 1 else (n - 1)
        return 2 * h.n_layers * per_ar * mc, 2 * h.n_layers * per_ar * (n - 1)

    @property
    def mega_active(self) -> bool:
        """True if the last single-token forward actually ran on the persistent kernel (it falls back per call when the shape or
        the co-residency check rules it out)."""
        return bool(self._lib.dl_engine_mega_active(self._h))

    def mega_vectors(self) -> dict:
        """The persistent kernel's phase vectors after its last launch, copied on the current stream: "x" (final residual),
        "qkv" (q|k|v before QK-norm and RoPE) and "z" (attention output) as (f32 payload, int64 epoch) pairs of LL words, and
        "h" (the last layer's SwiGLU output) as plain f32. Every vector carries its 8 tail words (zero unless overwritten)."""
        h = self.w.header
        n = {"x": h.dim, "qkv": self.qkv_dim, "z": self.w.n_heads * h.head_dim, "h": self.w.ff_dim}
        buf = {k: torch.empty((v + 8) * 2, dtype=torch.int32, device=self.device) for k, v in n.items()}
        cl.check(self._lib.dl_engine_mega_copy_vectors(self._h, *(buf[k].data_ptr() for k in ("x", "qkv", "z", "h")), cl.stream_ptr()),
                 "engine_mega_copy_vectors")
        out = {}
        for k in ("x", "qkv", "z"):
            words = buf[k].view(-1, 2)
            out[k] = (words[:, 0].view(torch.float32), words[:, 1].to(torch.int64) & 0xFFFFFFFF)
        out["h"] = buf["h"].view(torch.float32)
        return out

    def check_abort(self):
        """Raises if a device-side wait loop ran out of its spin budget (a peer rank died or a CTA never became resident): the
        kernels drain instead of hanging and flag the step as invalid (csrc/cuda/mega_decode.cu: SpinGuard)."""
        if self._lib.dl_engine_aborted(self._h):
            raise RuntimeError("device-side wait timed out: a tensor-parallel peer stopped responding (or the persistent kernel was not co-resident)")

    def enable_mega(self, enable: bool = True):
        """Single-token forwards through the persistent per-token kernel (dense models). The engine re-captures the decode graph."""
        cl.check(self._lib.dl_engine_enable_mega(self._h, 1 if enable else 0), "engine_enable_mega")
        self.mega = enable

    # -- tracing --
    def enable_trace(self, cap_launches: int = 1024, all_ctas: bool = False):
        """Device-side timeline: every kernel stamps globaltimer at entry / dependency resolved / prologue done / exit.
        The engine re-captures the decode graph with it. `all_ctas`: every CTA of the persistent kernel records its own
        phase stamps (row c of `trace_buf.view(num_sms, -1)`), for barrier-skew analysis."""
        if all_ctas:
            cap_launches = max(cap_launches, self.num_sms * 256)
        self.trace_buf = torch.zeros(cap_launches, 4, dtype=torch.int64, device=self.device)
        cl.check(self._lib.dl_engine_set_trace(self._h, self.trace_buf.data_ptr(), cap_launches), "engine_set_trace")
        cl.check(self._lib.dl_engine_set_trace_all(self._h, 1 if all_ctas else 0), "engine_set_trace_all")
        self.trace_stride = (cap_launches * 4) // self.num_sms if all_ctas else 0

    def read_trace(self):
        t = self.trace_buf.cpu().numpy()
        return t[t[:, 0] != 0]

    # -- low level --
    def _set_inputs(self, tokens: Sequence[int], start_pos: int):
        # Pageable source tensors: the copy is staged before the call returns, so back-to-back chunks cannot
        # overwrite a host buffer that an earlier async copy has not consumed yet.
        n = len(tokens)
        self.tokens[:n].copy_(torch.tensor(list(tokens), dtype=torch.int32))
        self.pos[:n].copy_(torch.arange(start_pos, start_pos + n, dtype=torch.int32))

    def forward_batch(self, tokens: Sequence[int], start_pos: int, logits_mode: int = 1, greedy_advance: bool = False):
        """Runs one forward over len(tokens) in {1,2,4,8} tokens at consecutive positions."""
        n = len(tokens)
        if start_pos + n > self.seq_len:
            raise ValueError("position beyond the context length")
        self._set_inputs(tokens, start_pos)
        self._forward(n, logits_mode, greedy_advance)

    def _forward(self, n: int, logits_mode: int, greedy_advance: bool = False):
        if self._parts:
            self._forward_parts(n, logits_mode, greedy_advance)
        else:
            cl.check(self._lib.dl_engine_forward(self._h, n, logits_mode, 1 if greedy_advance else 0, cl.stream_ptr()), "engine_forward")

    @property
    def tc_min_tokens(self) -> int:
        """Shortest prompt chunk the engine runs on the tensor-core GEMM path (default 9; 0: none). Shorter chunks run as GEMV batches."""
        return self._tc_min

    @tc_min_tokens.setter
    def tc_min_tokens(self, n: int) -> None:
        cl.check(self._lib.dl_engine_set_prefill_min_tc(self._h, int(n)), "engine_set_prefill_min_tc")
        self._tc_min = int(n)

    use_tc_prefill = property(lambda self: self._tc_min != 0, lambda self, on: setattr(self, "tc_min_tokens", 9 if on else 0))

    def prefill(self, tokens: Sequence[int], start_pos: int = 0, want_logits: bool = True) -> Optional[torch.Tensor]:
        """Feeds a prompt; returns the logits row of its last token (device tensor). The engine chunks it (dl_engine_prefill):
        up to max_prefill tokens a chunk on the tensor-core GEMM path, power-of-two GEMV batches otherwise. Library-collective
        tensor parallelism: GEMV batches of up to max_batch tokens with NCCL all-reduces."""
        tokens = list(tokens)
        if start_pos + len(tokens) > self.seq_len:
            raise ValueError("position beyond the context length")
        if not self._parts:
            self._prefill(tokens, start_pos, -1, want_logits)
            return self._full_logits(self.logits[0]) if want_logits else None
        for T, p, _ in prefill_plan(len(tokens), start_pos, self.seq_len, self.max_prefill, self.max_batch, 0, False):
            i = p - start_pos
            last = i + T == len(tokens)
            self.forward_batch(tokens[i:i + T], p, logits_mode=1 if (last and want_logits) else 0)
        return self._full_logits(self.logits[0]) if want_logits else None

    def prefill_plan(self, n: int, start_pos: int, slot: int = -1) -> List[tuple]:
        """The chunks prefill() (slot_prefill() for slot >= 0) runs for n tokens at start_pos with the engine's settings:
        (T, first position, on the tensor cores) per chunk."""
        if self._parts and slot < 0:
            return prefill_plan(n, start_pos, self.seq_len, self.max_prefill, self.max_batch, 0, False)
        return _plan_chunks(lambda out, cap: self._lib.dl_engine_prefill_plan(self._h, n, start_pos, slot, out, cap))

    def prefill_intermediates(self, rows: int, tensor_cores: bool) -> dict:
        """Copies of what the last prompt chunk of `rows` tokens left in the engine's scratch (its last layer). Tensor-core chunk:
        "x" (f32 residual), "qkv" (f32: q after QK-norm and RoPE, raw k and v), "xn" (bf16, the post-attention rmsnorm), "z" (bf16
        attention output), "h" (bf16 SwiGLU output). GEMV batch: "qkv", "z" and "h" in f32 (q is rotated in place for batches of
        2 or more); its residual is `x`."""
        w, hd = self.w, self.w.header.head_dim
        dims = {"x": w.header.dim, "qkv": self.qkv_dim, "xn": w.header.dim, "z": w.n_heads * hd, "h": w.ff_dim}
        keys = ("x", "qkv", "xn", "z", "h") if tensor_cores else ("qkv", "z", "h")
        dt = {"x": torch.float32, "qkv": torch.float32}
        out = {k: torch.empty(rows, dims[k], dtype=dt.get(k, torch.bfloat16 if tensor_cores else torch.float32), device=self.device)
               for k in keys}
        ptrs = [_p(out.get(k)) if tensor_cores else None for k in ("x", "qkv", "xn", "z", "h")]
        ptrs += [None if tensor_cores else _p(out[k]) for k in ("qkv", "z", "h")]
        cl.check(self._lib.dl_engine_prefill_scratch(self._h, rows, *ptrs, cl.stream_ptr()), "engine_prefill_scratch")
        return out

    def moe_intermediates(self, rows: int, tensor_cores: bool) -> dict:
        """The mixture-of-experts stages of the last prompt chunk of `rows` tokens (its last layer). Tensor-core chunk: "logits"
        (f32 router logits [rows][E]), "ids" (int32 [rows][k]), "weights" (f32 [rows][k]) and "h" (bf16 SwiGLU output of every
        (token, slot) pair [rows][k][ff]). One-token step (rows = 1): "logits" [E], "ids" and "weights" [k], "h" f32 [k][ff].
        The MoE rmsnorm output and the residual are "xn" and "x" of prefill_intermediates."""
        h, k, dev = self.w.header, self.w.header.n_active_experts, self.device
        lead = (rows,) if tensor_cores else ()
        out = {"logits": torch.empty(*lead, h.n_experts, dtype=torch.float32, device=dev),
               "ids": torch.empty(*lead, k, dtype=torch.int32, device=dev),
               "weights": torch.empty(*lead, k, dtype=torch.float32, device=dev),
               "h": torch.empty(*lead, k, self.w.ff_dim, dtype=torch.bfloat16 if tensor_cores else torch.float32, device=dev)}
        cl.check(self._lib.dl_engine_moe_scratch(self._h, rows, 1 if tensor_cores else 0, *(_p(out[n]) for n in ("logits", "ids", "weights", "h")),
                                                 cl.stream_ptr()), "engine_moe_scratch")
        return out

    def _prefill(self, tokens: List[int], start_pos: int, slot: int, want_logits: bool) -> None:
        arr = (C.c_int32 * len(tokens))(*tokens)
        cl.check(self._lib.dl_engine_prefill(self._h, arr, len(tokens), start_pos, slot, 1 if want_logits else 0, cl.stream_ptr()),
                 "engine_prefill")

    def step(self, token: int, pos: int) -> torch.Tensor:
        """Forward of one token; returns the full-vocabulary logits row (gathered over ranks under tensor parallelism)."""
        self.forward_batch([token], pos, logits_mode=1)
        return self._full_logits(self.logits[0])

    def _full_logits(self, local: torch.Tensor) -> torch.Tensor:
        if self.comm is None or self.comm.world_size == 1:
            return local
        return self.comm.all_gather_cat(local, dim=-1)

    def logits_all(self, tokens: Sequence[int], start_pos: int) -> torch.Tensor:
        """Logits for every token of a (<= max_batch, power of two) batch — used by perplexity and tests."""
        self.forward_batch(tokens, start_pos, logits_mode=2)
        return self._full_logits(self.logits[: len(tokens)])

    # -- library-collective path (tensor parallel): same kernels, all-reduce through torch.distributed between kernel groups --
    def _forward_parts(self, nb: int, logits_mode: int = 1, greedy_advance: bool = False) -> None:
        """One forward over the tokens staged in self.tokens/self.pos with per-layer NCCL all-reduces (the reference's K2/K3
        sync sites as library collectives, src/llm.cpp:397-403,548-554). Runs when the ranks do not share a peer-memory
        domain, for dense weight files, and as the baseline the fused kernels are measured against. Graph capturable."""
        import torch.distributed as dist
        y, sp, lib, h = self._ybuf, cl.stream_ptr(), self._lib, self._h
        tp = self.comm is not None and self.comm.world_size > 1
        cl.check(lib.dl_engine_forward_part(h, nb, 0, 0, y.data_ptr(), sp), "forward_part")
        for l in range(self.w.header.n_layers):
            for part in (1, 2):
                cl.check(lib.dl_engine_forward_part(h, nb, l, part, y.data_ptr(), sp), "forward_part")
                if tp:
                    dist.all_reduce(y[:nb])
                self.x[:nb].add_(y[:nb])
        if logits_mode:
            cl.check(lib.dl_engine_forward_part(h, nb, 0, 3 if logits_mode == 1 else 4, y.data_ptr(), sp), "forward_part")
        if greedy_advance:
            tok = self._full_logits(self.logits[0]).argmax().to(torch.int32).reshape(1)
            self.tokens[:1].copy_(tok)
            self.pos[:1].add_(1)
            self.history.index_copy_(0, self.pos[:1].long().clamp_(max=self.history.numel() - 1), tok)

    def forward_nccl_baseline(self, token_count: int = 1) -> torch.Tensor:
        """Library-collective forward of the staged tokens; returns the local logits slice (tools/bench_nccl_baseline.py)."""
        self._forward_parts(token_count, 1, False)
        return self.logits[0]

    # -- device-resident greedy decoding --
    def run_decode_step(self, use_graph: bool = True):
        """One greedy step on whatever (token, pos) currently sit in device memory; result lands in tokens[0]."""
        if self._parts:
            self._forward_parts(1, 1, True)
            return
        if use_graph:
            cl.check(self._lib.dl_engine_decode_graph(self._h, 1, cl.stream_ptr()), "engine_decode_graph")
        else:
            cl.check(self._lib.dl_engine_forward(self._h, 1, 1, 1, cl.stream_ptr()), "engine_forward")

    @property
    def launches_per_decode_step(self) -> int:
        if self.mega and self.mega_active:
            return 1                # one persistent kernel per token (plus a 4-byte memset node)
        if self._parts:
            return self.w.header.n_layers * 7 + 2
        if self.w.header.n_experts > 0:
            return self.w.header.n_layers * 6 + 2
        return self.w.header.n_layers * 5 + 2   # embedding + 5 fused kernels per layer + logits/arg-max

    @property
    def graph_captured(self) -> bool:
        """True while the engine holds a decode graph of its current configuration (captured on the first graph step)."""
        return bool(self._lib.dl_engine_graph_captured(self._h))

    # -- speculative decoding with a draft model (csrc/cuda/speculative.cu) --
    def spec_round(self, draft: "Engine", token: int, pos: int, k: int, use_graph: bool = True) -> tuple:
        """One round of greedy speculative decoding with this engine as the target: `token` is the last emitted token at `pos`,
        both engines hold valid KV rows for every position before it. The draft proposes k (1, 3 or 7; fewer near the end of the
        context) tokens, this engine checks them in one batched forward. Returns (emitted tokens, accepted drafts, drafts): the
        accepted drafts followed by this engine's own token after them, the tokens greedy decoding emits from (token, pos)."""
        out = (C.c_int32 * cl.SPEC_RESULT_WORDS)()
        cl.check(self._lib.dl_spec_round(self._h, draft._h, int(token), int(pos), int(k), 1 if use_graph else 0, out, cl.stream_ptr()),
                 "spec_round")
        n = out[1]
        return list(out[cl.SPEC_RESULT_HEAD:cl.SPEC_RESULT_HEAD + n]), int(out[0]), int(out[2])

    def verify(self, tokens: Sequence[int], start_pos: int) -> List[int]:
        """The verify forward of a speculative round over len(tokens) in {2, 4, 8} tokens at consecutive positions: logits of
        every row in logits[:n] and the arg-max of each row (lowest id among ties, ids at or above the vocabulary limit ignored)."""
        n = len(tokens)
        if start_pos + n > self.seq_len:
            raise ValueError("position beyond the context length")
        self._set_inputs(tokens, start_pos)
        out = (C.c_int32 * n)()
        cl.check(self._lib.dl_engine_verify(self._h, n, out, cl.stream_ptr()), "engine_verify")
        return list(out)

    def decode_greedy(self, first_token: int, start_pos: int, n_steps: int, use_graph: bool = True) -> List[int]:
        """Generates n_steps tokens greedily: step i consumes the token at position start_pos+i and emits the next.
        The loop runs entirely on the device (token + position live in device memory)."""
        if start_pos + n_steps > self.seq_len:
            raise ValueError("decode would run past the context length")
        self._set_inputs([first_token], start_pos)
        if self._parts:
            for _ in range(n_steps):
                self._forward_parts(1, 1, True)
        elif use_graph:
            cl.check(self._lib.dl_engine_decode_graph(self._h, n_steps, cl.stream_ptr()), "engine_decode_graph")
        else:
            for _ in range(n_steps):
                cl.check(self._lib.dl_engine_forward(self._h, 1, 1, 1, cl.stream_ptr()), "engine_forward")
        out = self.history[start_pos + 1: start_pos + 1 + n_steps].cpu()
        self.check_abort()
        return out.tolist()
