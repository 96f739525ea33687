"""Root/worker application runtime (reference: runInferenceApp / runWorkerApp, src/app.cpp:232-365).

Process model on a multi-GPU node: one process per GPU. Rank 0 is the *root* (tokenizer, sampler, user I/O), ranks >= 1 are
*workers*: they hold their tensor-parallel weight slices and mirror every forward the root issues. Control flows as the
reference's 8-byte LlmControlPacket {position, batchSize} (src/app.hpp:46-49) — here extended with an opcode and passed through a
shared-memory channel with heartbeats (parallel/control.py; torch.distributed broadcasts only when the ranks span hosts);
op 0 is the stop signal. All activation traffic happens inside the kernels over NVLink.
"""
from __future__ import annotations

import os
import sys
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from .. import host
from ..api import InferenceSession, check_logprobs
from .args import AppArgs

OP_STOP, OP_PREFILL, OP_STEP_LOGITS, OP_STEP_GREEDY, OP_DECODE_N, OP_STEP_SAMPLE, OP_SEED = 0, 1, 2, 3, 4, 5, 6
OP_CHOICES_SEED, OP_CHOICES_FIRST, OP_CHOICES_STEP = 7, 8, 9
OP_CONTROLS = 10   # [presence bits, frequency bits, count-row mask, (id, bias bits) ...]: Engine.set_sampling_controls
OP_FILTERS = 11    # [top_k, min_p bits]: Engine.set_sampling_filters


def _split_seed(seed: int) -> List[int]:
    return [seed & 0x7FFFFFFF, (seed >> 31) & 0x7FFFFFFF, (seed >> 62) & 0x3]


def _join_seed(w: Sequence[int]) -> int:
    return w[0] | (w[1] << 31) | (w[2] << 62)


def _active_mask(active: Sequence[bool]) -> int:
    return sum(1 << i for i, a in enumerate(active) if a)


def _active_list(mask: int, n: int) -> List[bool]:
    return [bool((mask >> i) & 1) for i in range(n)]


def _f32_bits(*xs: float) -> List[int]:
    import struct
    return list(struct.unpack(f"<{len(xs)}i", struct.pack(f"<{len(xs)}f", *xs)))


def _bits_f32(*xs: int) -> List[float]:
    import struct
    return list(struct.unpack(f"<{len(xs)}f", struct.pack(f"<{len(xs)}i", *xs)))


def _lp_kw(logprobs: Optional[int]) -> dict:
    return {} if logprobs is None else {"logprobs": logprobs}


def world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def init_distributed_from_env():
    """Initialises torch.distributed when launched by torchrun (RANK/WORLD_SIZE set). Returns (comm or None)."""
    ws = int(os.environ.get("WORLD_SIZE", "1"))
    if ws <= 1:
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        return None
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from ..parallel.comm import Communicator
    return Communicator()


def open_control_channel(comm):
    """Creates (rank 0) / attaches to (workers) the shared-memory control channel of the job. DL_CONTROL=nccl keeps the
    torch.distributed broadcasts (needed when the ranks do not share a host)."""
    if comm is None or os.environ.get("DL_CONTROL") == "nccl" or not getattr(comm, "single_node", True):
        return None
    import torch.distributed as dist
    from ..parallel.control import ControlChannel
    name = [None]
    chan = None
    if comm.rank == 0:
        chan = ControlChannel(0, comm.world_size)
        name[0] = chan.name
    dist.broadcast_object_list(name, src=0)
    if comm.rank != 0:
        chan = ControlChannel(comm.rank, comm.world_size, name=name[0])
    chan.start_heartbeat()
    dist.barrier()
    return chan


class RootInference:
    """Root-side handle (reference RootLlmInference, src/app.cpp:168-208): every call first tells the workers what to run.
    The packet travels through shared memory (parallel/control.py); the activations never leave the GPUs."""

    def __init__(self, sess: InferenceSession, comm, chan=None):
        self.sess = sess
        self.comm = comm
        self.chan = chan
        self.eng = sess.engine
        self.header = sess.header
        self.eval_ms = 0.0
        self._ctl = torch.zeros(4, dtype=torch.int64, device=sess.device) if (comm is not None and chan is None) else None
        on_gpu = torch.device(sess.device).type == "cuda"   # the session's device, not whether the machine has a GPU
        self._pin_out = torch.zeros(1, dtype=torch.int32).pin_memory() if on_gpu else None
        self._pin_in = torch.zeros(2, dtype=torch.int32).pin_memory() if on_gpu else None

    def _send(self, op: int, pos: int, tokens: Sequence[int]):
        if self.comm is None:
            return
        if self.chan is not None:
            self.chan.send(op, pos, tokens)
            return
        import torch.distributed as dist
        n = len(tokens)
        self._ctl[0], self._ctl[1], self._ctl[2] = op, pos, n
        dist.broadcast(self._ctl, 0)
        if n:
            t = torch.tensor(list(tokens), dtype=torch.int64, device=self.sess.device)
            dist.broadcast(t, 0)

    def prefill(self, tokens: Sequence[int], pos: int) -> None:
        if tokens:
            self._send(OP_PREFILL, pos, tokens)
            self.eng.prefill(tokens, pos, want_logits=False)

    def forward_logits(self, token: int, pos: int) -> torch.Tensor:
        self._send(OP_STEP_LOGITS, pos, [token])
        return self.eng.step(token, pos)

    def forward_greedy(self, token: int, pos: int, logprobs: Optional[int] = None) -> int:
        self._send(OP_STEP_GREEDY, pos, [token])
        if self._pin_in is None:          # session on the CPU (protocol tests)
            self.eng._set_inputs([token], pos)
            self.eng.run_decode_step()
            return int(self.eng.tokens[0])
        # the root synchronises every step, so one pinned staging slot is enough (workers enqueue ahead: pageable staging)
        self._pin_in[0], self._pin_in[1] = token, pos
        self.eng.tokens[:1].copy_(self._pin_in[:1], non_blocking=True)
        self.eng.pos[:1].copy_(self._pin_in[1:2], non_blocking=True)
        self.eng.run_decode_step()
        lp = logprobs
        if lp is not None:
            self.eng.logprobs([lp])
        self._pin_out.copy_(self.eng.tokens[:1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.eng.check_abort()
        if lp is not None:
            self._last_logprobs = self.eng.read_logprobs()
        return int(self._pin_out[0])

    # ---- sampling on the device: the logits never leave the GPUs (csrc/cuda/sampler.cu) ----
    @property
    def device_sampling(self) -> bool:
        return self._pin_in is not None and not getattr(self.eng, "_parts", False) and os.environ.get("DL_HOST_SAMPLER") is None

    def seed(self, seed: int) -> None:
        self._send(OP_SEED, 0, _split_seed(seed))
        self.eng.seed_sampler(seed)

    def forward_sampled(self, token: int, pos: int, temperature: float, topp: float, logprobs: Optional[int] = None) -> int:
        import struct
        t_bits, p_bits = struct.unpack("<ii", struct.pack("<ff", temperature, topp))
        self._send(OP_STEP_SAMPLE, pos, [token, t_bits, p_bits])
        self.eng.step_sampled(token, pos, temperature, topp)
        lp = logprobs
        if lp is not None:
            self.eng.logprobs([lp], controlled=True)
        self._pin_out.copy_(self.eng.tokens[:1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.eng.check_abort()
        if lp is not None:
            self._last_logprobs = self.eng.read_logprobs()
        return int(self._pin_out[0])

    def set_controls(self, sampler, row_mask: int) -> None:
        bias = sampler.logit_bias
        words = _f32_bits(sampler.presence_penalty, sampler.frequency_penalty) + [row_mask]
        for t, v in bias:
            words += [t] + _f32_bits(v)
        self._send(OP_CONTROLS, 0, words)
        self.eng.set_sampling_controls(sampler.presence_penalty, sampler.frequency_penalty, bias, row_mask)

    def set_filters(self, sampler) -> None:
        """The sampler's top_k / min_p on every rank, before the first draw that uses them (each rank draws from the gathered
        logits with its own generator, so all ranks must hold the same filters)."""
        key = (sampler.top_k, sampler.min_p)
        if getattr(self, "_filters", (0, 0.0)) != key:
            self._send(OP_FILTERS, 0, [key[0]] + _f32_bits(key[1]))
            self.eng.set_sampling_filters(*key)
            self._filters = key

    def next_token(self, token: int, pos: int, sampler, logprobs: Optional[int] = None) -> int:
        """One generated token with the sampler's settings: greedy and temperature/top-p both run on the device; the host sampler
        is only used with the library-collective (multi-node) mode or DL_HOST_SAMPLER=1. Greedy with sampling controls runs
        on the device sampler (arg-max of the controlled logits), not on the fused arg-max. logprobs = k: also the
        log-probabilities of the draw on the device (last_logprobs(); one GPU only), enqueued behind it."""
        if logprobs is not None:
            check_logprobs(logprobs, self.comm.world_size if self.comm is not None else 1)
        if sampler.temperature == 0.0 and not sampler.controls_active:
            return self.forward_greedy(token, pos, logprobs)
        if self.device_sampling:
            if sampler.temperature != 0.0 and getattr(self, "_seeded", None) != (sampler.seed, sampler.seed_generation):
                self.seed(sampler.seed)
                self._seeded = (sampler.seed, sampler.seed_generation)
            key = sampler.completion_generation if sampler.controls_active else None
            if getattr(self, "_controls", None) != key:   # a new completion: count row 0 starts from zero
                self.set_controls(sampler, 1)
                self._controls = key
            self.set_filters(sampler)
            return self.forward_sampled(token, pos, sampler.temperature, sampler.topp, logprobs)
        t = int(sampler.sample(self.forward_logits(token, pos).float().cpu().numpy()))
        if logprobs is not None:
            self._last_logprobs = [self.eng.logprobs_host_draw(t, logprobs, sampler)]
        return t

    def last_logprobs(self) -> list:
        """The log-probability entries of the last next_token / choices call asked for them (InferenceSession.last_logprobs)."""
        return self._last_logprobs

    # ---- several completions of one prompt (api.run_choices); workers mirror every batched step ----
    def forget_device_seed(self):
        self._seeded = None

    def save_sampler(self):
        key = getattr(self, "_seeded", None)
        return key, (self.eng.sampler_state() if key is not None and self.device_sampling else 0)

    def restore_sampler(self, saved):
        key, state = saved
        if key is not None and self.device_sampling:
            self.seed(state)
        self._seeded = key

    def batched_choices(self, n: int) -> bool:
        return self.device_sampling and self.eng.supports_choices(n)

    def choice_controls(self, sampler, n: int) -> None:
        self.set_filters(sampler)
        if sampler.controls_active or getattr(self, "_controls", None) is not None:
            self.set_controls(sampler, ((1 << n) - 1) << 1)
            self._controls = -1 if sampler.controls_active else None   # row 0's counts are not this sampler's

    def seed_choices(self, seeds: Sequence[int]) -> None:
        self._send(OP_CHOICES_SEED, 0, [w for s in seeds for w in _split_seed(s)])
        self.eng.seed_choice_samplers(seeds)

    def choices_first(self, token: int, P: int, n: int, temperature: float, topp: float, logprobs: Optional[int] = None) -> List[int]:
        self._send(OP_CHOICES_FIRST, P, [token, n] + _f32_bits(temperature, topp))
        out = self.eng.choices_first(token, P, n, temperature, topp, **_lp_kw(logprobs))
        if logprobs is not None:
            self._last_logprobs = self.eng.read_logprobs()
        return out

    def choices_step(self, tokens: Sequence[int], P: int, C: int, j: int, active: Sequence[bool], temperature: float,
                     topp: float, logprobs: Optional[int] = None) -> List[int]:
        self._send(OP_CHOICES_STEP, P, [C, j, _active_mask(active)] + _f32_bits(temperature, topp) + list(tokens))
        out = self.eng.choices_step(tokens, P, C, j, active, temperature, topp, **_lp_kw(logprobs))
        if logprobs is not None:
            self._last_logprobs = self.eng.read_logprobs()
        return out

    def decode_greedy(self, token: int, pos: int, n_steps: int) -> List[int]:
        """n greedy steps with the token fed back on the device (no host round trip per step): one control packet for all."""
        self._send(OP_DECODE_N, pos, [token, n_steps])
        return self.eng.decode_greedy(token, pos, n_steps)

    def finish(self):
        try:
            self._send(OP_STOP, 0, [])
        finally:
            if self.chan is not None:
                self.chan.close()


def worker_loop(sess: InferenceSession, comm, chan=None) -> None:
    """Worker main loop (reference runWorkerApp, src/app.cpp:306-365): mirror the root's forwards until the stop packet."""
    import torch.distributed as dist
    ctl = torch.zeros(4, dtype=torch.int64, device=sess.device) if chan is None else None
    eng = sess.engine
    while True:
        if chan is not None:
            op, pos, toks = chan.recv()
        else:
            dist.broadcast(ctl, 0)
            op, pos, n = int(ctl[0]), int(ctl[1]), int(ctl[2])
            toks = []
            if op != OP_STOP and n:
                t = torch.zeros(n, dtype=torch.int64, device=sess.device)
                dist.broadcast(t, 0)
                toks = t.tolist()
        if op == OP_STOP:
            print("🛑 Stop signal")
            if chan is not None:
                chan.close()
            return
        if op == OP_PREFILL:
            eng.prefill(toks, pos, want_logits=False)
        elif op == OP_STEP_LOGITS:
            eng.step(toks[0], pos)
        elif op == OP_STEP_GREEDY:
            eng._set_inputs(toks, pos)
            eng.run_decode_step()
        elif op == OP_DECODE_N:
            eng.decode_greedy(toks[0], pos, toks[1])
        elif op == OP_SEED:
            eng.seed_sampler(_join_seed(toks))
        elif op == OP_CHOICES_SEED:
            eng.seed_choice_samplers([_join_seed(toks[i:i + 3]) for i in range(0, len(toks), 3)])
        elif op == OP_CHOICES_FIRST:
            temperature, topp = _bits_f32(toks[2], toks[3])
            eng.choices_first(toks[0], pos, toks[1], temperature, topp)
        elif op == OP_CHOICES_STEP:
            C, j, mask = toks[0], toks[1], toks[2]
            temperature, topp = _bits_f32(toks[3], toks[4])
            tokens = toks[5:]
            eng.choices_step(tokens, pos, C, j, _active_list(mask, len(tokens)), temperature, topp)
        elif op == OP_CONTROLS:
            presence, frequency = _bits_f32(toks[0], toks[1])
            pairs = toks[3:]
            bias = [(pairs[i], _bits_f32(pairs[i + 1])[0]) for i in range(0, len(pairs), 2)]
            eng.set_sampling_controls(presence, frequency, bias, toks[2])
        elif op == OP_FILTERS:
            eng.set_sampling_filters(toks[0], _bits_f32(toks[1])[0])
        elif op == OP_STEP_SAMPLE:
            import struct
            temperature, topp = struct.unpack("<ff", struct.pack("<ii", toks[1], toks[2]))
            eng.step_sampled(toks[0], pos, temperature, topp)


def kv_cache_bytes(header, n_ranks: int, kv_type: str) -> int:
    """Device bytes of one rank's K and V caches: bf16 = 2 bytes a value, q80 = 1 byte a value + a 2-byte scale per 32."""
    kv_heads = header.n_kv_heads // n_ranks if header.n_kv_heads >= n_ranks else 1
    values = 2 * header.n_layers * header.seq_len * kv_heads * header.head_dim
    return values * 2 if kv_type == "bf16" else values + values // 16


@dataclass
class AppContext:
    args: AppArgs
    sess: InferenceSession
    inference: RootInference
    tokenizer: object
    sampler: object
    header: object


def run_inference_app(args: AppArgs, handler: Callable[[AppContext], None]) -> None:
    if args.model is None:
        raise RuntimeError("Model is required")
    if args.tokenizer is None:
        raise RuntimeError("Tokenizer is required")
    comm = init_distributed_from_env()
    rank = comm.rank if comm else 0
    H = host()
    header = H.load_model_header(args.model, args.max_seq_len)
    n_nodes = comm.world_size if comm else 1
    if header.weight_type == H.F_Q40 and args.buffer_float_type != "q80":
        raise RuntimeError("This version supports only Q40 weights with Q80 sync type")
    sess = InferenceSession(args.model, args.tokenizer, max_seq_len=args.max_seq_len, temperature=args.temperature,
                            topp=args.topp, seed=args.seed, comm=comm, moe_mode=getattr(args, "moe_mode", "auto") or "auto",
                            presence_penalty=args.presence_penalty, frequency_penalty=args.frequency_penalty,
                            parallel=getattr(args, "parallel", 1), kv_cache_float_type=args.kv_cache_float_type,
                            top_k=getattr(args, "top_k", 0), min_p=getattr(args, "min_p", 0.0))
    chan = open_control_channel(comm)
    if rank != 0:
        worker_loop(sess, comm, chan)
        return
    tok = sess.tokenizer
    if args.info:
        if tok.vocab_size != header.vocab_size:
            print(f"Tokenizer vocab size ({tok.vocab_size}) does not match the model vocab size ({header.vocab_size})")
        print(tok.describe(), end="")
        print(header.describe(), end="")
        req = H.required_device_bytes(header, n_nodes, 0) + kv_cache_bytes(header, n_nodes, args.kv_cache_float_type)
        print(f"📀 RequiredMemory: {req // (1024 * 1024)} MB")
        name = torch.cuda.get_device_name(sess.device)
        print(f"🧠 GPU: {name} x{n_nodes} (sm_90a kernels; tensor parallel over NVLink peer memory)")
        print("💿 Weights loaded")
    inf = RootInference(sess, comm, chan)
    ctx = AppContext(args=args, sess=sess, inference=inf, tokenizer=tok, sampler=sess.sampler, header=header)
    try:
        handler(ctx)
    finally:
        inf.finish()
