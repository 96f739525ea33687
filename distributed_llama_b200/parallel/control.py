"""Root -> worker control channel through POSIX shared memory, with liveness tracking.

Reference counterpart: the 8-byte LlmControlPacket {position, batchSize} the root writes to every worker socket before each
forward (src/app.hpp:46-49, src/app.cpp:197-230), the worker's polling loop with its busy/blocking modes (src/app.cpp:332-363)
and the socket exceptions that end a session when a peer disappears (src/nn/nn-network.cpp:84-123, src/app.cpp:356-362).

All ranks of a job are processes on one box (one per GPU), so the packet does not need a network: the root writes
{op, pos, n, tokens[n]} into a shared segment and bumps a sequence number; workers spin on that number (sub-microsecond
hand-off instead of two NCCL broadcasts + a device sync per token), fall back to sleeping polls after a second of idleness
(the reference's "turbo off" mode), acknowledge each packet, and publish a heartbeat. A peer whose heartbeat goes stale — or a
worker that stops acknowledging — surfaces as `PeerLost` on the other side instead of a hang.
"""
from __future__ import annotations

import os
import struct
import time
from multiprocessing import shared_memory
from typing import List, Optional, Sequence, Tuple

import numpy as np

MAX_TOKENS = 8192
_HDR_WORDS = 64          # u64 words: [0] seq, [1] op, [2] pos, [3] n, [8..16) ack per rank, [16..24) heartbeat per rank (ns)
_ACK0, _HB0 = 8, 16

# The packets: op, position and int32 words. The root sends them before every engine call a worker must repeat
# (api.TokenSteps._send, apps.runtime.RootInference); apps.runtime.worker_loop makes the same call.
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
    return list(struct.unpack(f"<{len(xs)}i", struct.pack(f"<{len(xs)}f", *xs)))


def _bits_f32(*xs: int) -> List[float]:
    return list(struct.unpack(f"<{len(xs)}f", struct.pack(f"<{len(xs)}i", *xs)))


class PeerLost(RuntimeError):
    """A rank of the job stopped responding (process died or its GPU wedged)."""


def _now_ns() -> int:
    return time.monotonic_ns()


class ControlChannel:
    def __init__(self, rank: int, world_size: int, name: Optional[str] = None, timeout_s: Optional[float] = None):
        """Rank 0 creates the segment (name=None) and must hand `self.name` to the workers (any out-of-band way: the launcher
        passes it through torch.distributed or the environment); workers attach by name."""
        self.rank, self.world = rank, world_size
        self.timeout_ns = int(1e9 * (timeout_s if timeout_s is not None else float(os.environ.get("DL_PEER_TIMEOUT", "60"))))
        size = _HDR_WORDS * 8 + MAX_TOKENS * 4
        if rank == 0:
            self.shm = shared_memory.SharedMemory(create=True, size=size, name=name)
            self.shm.buf[:size] = bytes(size)
        else:
            assert name is not None
            self.shm = shared_memory.SharedMemory(name=name)
            try:   # the creator unlinks; attaching processes must not let the resource tracker remove the segment at exit
                from multiprocessing import resource_tracker
                resource_tracker.unregister(self.shm._name, "shared_memory")
            except Exception:
                pass
        self.name = self.shm.name
        self.hdr = np.ndarray((_HDR_WORDS,), dtype=np.uint64, buffer=self.shm.buf)
        self.tok = np.ndarray((MAX_TOKENS,), dtype=np.int32, buffer=self.shm.buf, offset=_HDR_WORDS * 8)
        self.seq = 0      # a fresh channel starts at packet 0; a worker that attaches late still sees packet 1 (the root waits for its ack)
        self._hb_thread = None
        self.beat()

    # ---- liveness ----
    def start_heartbeat(self, period_s: float = 0.5) -> None:
        """Background heartbeat: keeps this rank 'alive' for its peers while the main thread blocks (user input, long loads)."""
        import threading

        def run():
            while self.hdr is not None:
                try:
                    self.beat()
                except Exception:
                    return
                time.sleep(period_s)
        self._hb_thread = threading.Thread(target=run, daemon=True)
        self._hb_thread.start()

    def beat(self) -> None:
        self.hdr[_HB0 + self.rank] = _now_ns()

    def stale_ranks(self, ranks: Sequence[int]) -> List[int]:
        now = _now_ns()
        return [r for r in ranks if now - int(self.hdr[_HB0 + r]) > self.timeout_ns]

    # ---- root side ----
    def send(self, op: int, pos: int, tokens: Sequence[int] = ()) -> None:
        """Publishes one packet. Blocks until every worker has consumed the previous one."""
        n = len(tokens)
        if n > MAX_TOKENS:
            raise ValueError("control packet too large")
        self.wait_acks()
        if n:
            self.tok[:n] = np.asarray(tokens, dtype=np.int32)
        self.hdr[1], self.hdr[2], self.hdr[3] = op, pos, n
        self.seq += 1
        self.hdr[0] = self.seq            # published last: the payload above is complete when a reader sees the new number
        self.beat()

    def wait_acks(self) -> None:
        workers = range(1, self.world)
        spins = 0
        t0 = None
        while True:
            if all(int(self.hdr[_ACK0 + r]) >= self.seq for r in workers):
                return
            spins += 1
            if spins & 0xFFF == 0:
                self.beat()
                now = _now_ns()
                t0 = t0 or now
                if now - t0 > self.timeout_ns:
                    behind = [r for r in workers if int(self.hdr[_ACK0 + r]) < self.seq]
                    raise PeerLost(f"worker rank(s) {behind} did not acknowledge control packet {self.seq}")
                if now - t0 > 1_000_000_000:
                    time.sleep(0.001)

    # ---- worker side ----
    def recv(self) -> Tuple[int, int, List[int]]:
        """Waits for the next packet; returns (op, pos, tokens). Busy-polls for a second, then sleeps between polls (reference
        worker: non-blocking sockets while busy, blocking after 1 s idle)."""
        spins = 0
        t_idle = None
        while int(self.hdr[0]) == self.seq:
            spins += 1
            if spins & 0x3FF == 0:
                self.beat()
                now = _now_ns()
                t_idle = t_idle or now
                if now - int(self.hdr[_HB0]) > self.timeout_ns:
                    raise PeerLost("the root stopped sending heartbeats")
                if now - t_idle > 1_000_000_000:
                    time.sleep(0.002)
        self.seq = int(self.hdr[0])
        op, pos, n = int(self.hdr[1]), int(self.hdr[2]), int(self.hdr[3])
        toks = self.tok[:n].tolist()
        self.hdr[_ACK0 + self.rank] = self.seq
        self.beat()
        return op, pos, toks

    def close(self) -> None:
        try:
            self.hdr = None
            self.tok = None
            self.shm.close()
            if self.rank == 0:
                self.shm.unlink()
        except Exception:
            pass
