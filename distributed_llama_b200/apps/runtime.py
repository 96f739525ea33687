"""Root/worker application runtime (reference: runInferenceApp / runWorkerApp, src/app.cpp:232-365).

Process model on a multi-GPU node: one process per GPU. Rank 0 is the *root* (tokenizer, sampler, user I/O), ranks >= 1 are
*workers*: they hold their tensor-parallel weight slices and mirror every forward the root issues. Control flows as the
reference's 8-byte LlmControlPacket {position, batchSize} (src/app.hpp:46-49) — here extended with an opcode and passed through a
shared-memory channel with heartbeats (parallel/control.py; torch.distributed broadcasts only when the ranks span hosts);
op 0 is the stop signal. All activation traffic happens inside the kernels over NVLink.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Callable, Sequence

import torch

from .. import host
from ..api import InferenceSession, TokenSteps
# the packet format; the op codes and word helpers also stay importable from this module (_f32_bits: encoding only)
from ..parallel.control import (OP_CHOICES_FIRST, OP_CHOICES_SEED, OP_CHOICES_STEP, OP_CONTROLS, OP_DECODE_N, OP_FILTERS,  # noqa: F401
                                OP_PREFILL, OP_SEED, OP_STEP_GREEDY, OP_STEP_LOGITS, OP_STEP_SAMPLE, OP_STOP, _active_list,
                                _bits_f32, _f32_bits, _join_seed)
from .args import AppArgs


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


class RootInference(TokenSteps):
    """Root-side handle (reference RootLlmInference, src/app.cpp:168-208): the token steps of api.TokenSteps over the session's
    engine, every engine call first announced to the workers. The packet travels through shared memory (parallel/control.py),
    or torch.distributed broadcasts without a channel; the activations never leave the GPUs."""

    def __init__(self, sess: InferenceSession, comm, chan=None):
        super().__init__(sess.engine, sess.device, comm.world_size if comm is not None else 1,
                         getattr(sess, "draft", None), getattr(sess, "draft_tokens", 3))
        self.comm = comm
        self.chan = chan
        self._ctl = torch.zeros(4, dtype=torch.int64, device=self.device) if (comm is not None and chan is None) else None

    def _send(self, op: int, pos: int, words: Sequence[int]) -> None:
        if self.comm is None:
            return
        if self.chan is not None:
            self.chan.send(op, pos, words)
            return
        import torch.distributed as dist
        n = len(words)
        self._ctl[0], self._ctl[1], self._ctl[2] = op, pos, n
        dist.broadcast(self._ctl, 0)
        if n:
            t = torch.tensor(list(words), dtype=torch.int64, device=self.device)
            dist.broadcast(t, 0)

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
            temperature, topp = _bits_f32(toks[1], toks[2])
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
                            parallel=getattr(args, "parallel", 1), parallel_cache=getattr(args, "parallel_cache", "split"),
                            kv_cache_float_type=args.kv_cache_float_type,
                            top_k=getattr(args, "top_k", 0), min_p=getattr(args, "min_p", 0.0),
                            draft_model=args.draft_model, draft_tokens=args.draft_tokens)
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
