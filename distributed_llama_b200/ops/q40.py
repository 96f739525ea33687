"""Device-side q40 matrices: repack from `.m` bytes and the standalone GEMV entry point (tests, microbenchmarks)."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional

import torch

from . import cuda_lib as cl


@dataclass
class DeviceQ40:
    """q40 matrix in the device layout of csrc/cuda/common.cuh: qs u32 [d][n/8], scales f16 [d][n/32]."""
    qs: torch.Tensor
    scales: torch.Tensor
    d: int
    n: int

    @staticmethod
    def empty(d: int, n: int, device="cuda", lead: int = 1) -> "DeviceQ40":
        qs = torch.empty((lead * d, n // 8), dtype=torch.int32, device=device)
        sc = torch.empty((lead * d, n // 32), dtype=torch.float16, device=device)
        return DeviceQ40(qs, sc, d, n)

    def to_f32(self) -> torch.Tensor:
        rows = self.qs.shape[0]
        out = torch.empty((rows, self.n), dtype=torch.float32, device=self.qs.device)
        cl.check(cl.lib().dl_dequant_device_q40(self.qs.data_ptr(), self.scales.data_ptr(), rows, self.n // 32,
                                                 out.data_ptr(), cl.stream_ptr()), "dequant_device_q40")
        return out


@dataclass
class DeviceDense:
    """Row-major f32 / f16 matrix [lead*d][n] for `.m` files that are not q40 (csrc/cuda/gemv_dense.cu). Exposes the same
    `qs` / `scales` attributes as DeviceQ40 so the engine's pointer tables do not care which kind they carry."""
    data: torch.Tensor
    d: int
    n: int

    @property
    def qs(self) -> torch.Tensor:
        return self.data

    @property
    def scales(self):
        return None

    @property
    def wtype(self) -> int:
        return 1 if self.data.dtype == torch.float32 else 2

    def to_f32(self) -> torch.Tensor:
        return self.data.float()


def gemv_dense(w: DeviceDense, x: torch.Tensor, *, pro: int, epi: int, out: torch.Tensor, norm_w: Optional[torch.Tensor] = None,
               eps: float = 1e-5, num_sms: int = 0, pdl: bool = False, act_fn: int = 0) -> torch.Tensor:
    """Dense-weight counterpart of gemv_q40 (f32 activations, no q80 round trip)."""
    nb = x.shape[0]
    if num_sms == 0:
        num_sms = torch.cuda.get_device_properties(x.device).multi_processor_count
    cl.check(cl.lib().dl_gemv_dense(w.wtype, pro, epi, nb, w.data.data_ptr(), w.d, w.n, x.data_ptr(), x.stride(0),
                                    norm_w.data_ptr() if norm_w is not None else None, eps, out.data_ptr(), out.stride(0),
                                    num_sms, cl.stream_ptr(), 1 if pdl else 0, act_fn), "gemv_dense")
    return out


def gemv_dense_smem_bytes(d: int, n: int, nb: int, num_sms: int) -> int:
    """Shared memory of a dense GEMV launch of nb tokens over a [d][n] matrix; the kernel refuses more than 227 KB."""
    return cl.lib().dl_gemv_dense_smem_bytes(d, n, nb, num_sms)


def repack_q40(raw: torch.Tensor, rows: int, n_cols: int, dst: DeviceQ40, *, src_row_pitch: Optional[int] = None,
               src_col_byte_offset: int = 0, dst_row_stride: int = 1, dst_row_offset: int = 0, head_dim: int = 0) -> None:
    """raw: uint8 CUDA tensor holding `rows` source rows of 18-byte blocks (pitch defaults to n_cols/32*18)."""
    assert raw.is_cuda and raw.dtype == torch.uint8
    bpr = n_cols // 32
    pitch = src_row_pitch if src_row_pitch is not None else bpr * 18
    assert dst.n == n_cols
    cl.check(cl.lib().dl_repack_q40(raw.data_ptr(), pitch, src_col_byte_offset, rows, bpr, dst.qs.data_ptr(),
                                    dst.scales.data_ptr(), dst_row_stride, dst_row_offset, head_dim, cl.stream_ptr()),
             "repack_q40")


GEMV_IMPLS = {"auto": 0, "ldg": 1, "tma": 2}


def gemv_q40(w: DeviceQ40, x: torch.Tensor, *, pro: int, epi: int, out: torch.Tensor, norm_w: Optional[torch.Tensor] = None,
             eps: float = 1e-5, num_sms: int = 0, pdl: bool = False, impl: str = "auto", act_fn: int = 0) -> torch.Tensor:
    """x: f32 [nb, n]; out: f32 [nb, d] (STORE / RESIDUAL in place) or [nb, d/2] (SWIGLU). impl "tma" raises (code 1) when the
    shape does not fit the TMA kernel. act_fn: gate activation of the SwiGLU epilogue (0 = SiLU, 1 = tanh-GELU)."""
    nb = x.shape[0]
    if num_sms == 0:
        num_sms = torch.cuda.get_device_properties(x.device).multi_processor_count
    cl.check(cl.lib().dl_gemv_q40(pro, epi, nb, w.qs.data_ptr(), w.scales.data_ptr(), w.d, w.n, x.data_ptr(), x.stride(0),
                                  norm_w.data_ptr() if norm_w is not None else None, eps, out.data_ptr(), out.stride(0),
                                  num_sms, cl.stream_ptr(), 1 if pdl else 0, GEMV_IMPLS[impl], act_fn), "gemv_q40")
    return out


@dataclass(frozen=True)
class GemvPlan:
    """What gemv_q40 runs for a one-rank launch (dl_gemv_q40_plan). kernel: 1 per-thread loads ("ldg"), 2 TMA ring ("tma");
    stage_rows / n_stages: the ring (0 for kernel 1); launches > 1: the batch runs as that many launches of nb / launches tokens,
    the other fields describing one of them. rc 1: impl "tma" and the shape does not fit it; rc < 0: refused."""
    rc: int
    kernel: int
    grid: int
    max_tile_rows: int
    stage_rows: int
    n_stages: int
    smem_bytes: int
    launches: int


def gemv_q40_plan(pro: int, epi: int, nb: int, d: int, n: int, *, num_sms: int, impl: str = "auto") -> GemvPlan:
    """The dispatch decision of gemv_q40; launches nothing."""
    out = (ctypes.c_int * 8)()
    cl.lib().dl_gemv_q40_plan(pro, epi, nb, d, n, num_sms, GEMV_IMPLS[impl], out)
    return GemvPlan(*out)


def gemv_q40_argmax(w: DeviceQ40, x: torch.Tensor, *, norm_w: torch.Tensor, eps: float, out: torch.Tensor, arg_val: torch.Tensor,
                    arg_idx: torch.Tensor, arg_counter: torch.Tensor, token: torch.Tensor, pos: torch.Tensor,
                    history: Optional[torch.Tensor], history_cap: int, row_offset: int = 0, vocab_limit: int = 0,
                    num_sms: int = 0) -> None:
    """Fused logits + greedy token of one token on the TMA kernel: out [d] = logits of rmsnorm(x) [n]; token[0] = lowest-index
    maximum among rows with row_offset + r < vocab_limit (0: all); pos[0] += 1; history[pos] = token while pos < history_cap.
    arg_val / arg_idx: one entry per CTA; arg_counter: zero, left at zero."""
    if num_sms == 0:
        num_sms = torch.cuda.get_device_properties(x.device).multi_processor_count
    cl.check(cl.lib().dl_gemv_q40_argmax(w.qs.data_ptr(), w.scales.data_ptr(), w.d, w.n, x.data_ptr(), norm_w.data_ptr(), eps, out.data_ptr(),
                                         arg_val.data_ptr(), arg_idx.data_ptr(), arg_counter.data_ptr(), token.data_ptr(), pos.data_ptr(),
                                         history.data_ptr() if history is not None else None, history_cap, row_offset, vocab_limit,
                                         num_sms, cl.stream_ptr()), "gemv_q40_argmax")


def argmax_advance(logits: torch.Tensor, vocab: int, token: torch.Tensor, pos: torch.Tensor, history: Optional[torch.Tensor],
                   history_cap: int) -> None:
    """Stand-alone greedy token: token[0] = lowest index among the maxima of logits[:vocab]; pos[0] += 1; history[pos] = token
    while pos < history_cap."""
    cl.check(cl.lib().dl_argmax_advance(logits.data_ptr(), vocab, token.data_ptr(), pos.data_ptr(),
                                        history.data_ptr() if history is not None else None, history_cap, cl.stream_ptr()),
             "argmax_advance")


GEMM_VARIANTS = {"auto": 0, "ldg": 1, "tma": 2}


def gemm_q40_tc(w: DeviceQ40, act: torch.Tensor, *, epi: int, out: torch.Tensor, num_sms: int = 0, pdl: bool = False,
                variant: str = "auto", act_fn: int = 0) -> torch.Tensor:
    """Tensor-core (wgmma) prefill GEMM. act: bf16 [T, n] (T <= 256); out: [T, d] f32 (STORE/RESIDUAL), bf16 [T, d/2] (SWIGLU) or bf16 [T, d].
    act_fn: gate activation of the SwiGLU epilogue (0 = SiLU, 1 = tanh-GELU)."""
    assert act.dtype == torch.bfloat16 and act.is_cuda and act.stride(1) == 1
    if num_sms == 0:
        num_sms = torch.cuda.get_device_properties(act.device).multi_processor_count
    cl.check(cl.lib().dl_gemm_q40_tc(epi, w.qs.data_ptr(), w.scales.data_ptr(), w.d, w.n, act.data_ptr(), act.stride(0), act.shape[0],
                                     out.data_ptr(), out.stride(0), num_sms, act_fn, cl.stream_ptr(), 1 if pdl else 0,
                                     GEMM_VARIANTS[variant]), "gemm_q40_tc")
    return out


@dataclass(frozen=True)
class GemmPlan:
    """What gemm_q40_tc runs for a shape (dl_gemm_q40_tc_plan). kernel: 1 register-prefetch ("ldg"), 2 TMA-staged ("tma");
    split_k > 1 with cluster = 1: partial sums reduced inside a thread-block cluster, cluster = 0: through the global scratch."""
    rc: int
    kernel: int
    split_k: int
    cluster: int
    grid: int
    stages: int
    raw_stages: int
    b_stages: int


def gemm_q40_tc_plan(epi: int, d: int, n: int, T: int, *, act_stride: Optional[int] = None, num_sms: int, variant: str = "auto") -> GemmPlan:
    """The dispatch decision of gemm_q40_tc (reads DL_GEMM_CLUSTER / DL_GEMM_SPLITK like the launch); launches nothing."""
    out = (ctypes.c_int * 8)()
    cl.lib().dl_gemm_q40_tc_plan(epi, d, n, T, n if act_stride is None else act_stride, num_sms, GEMM_VARIANTS[variant], out)
    return GemmPlan(*out)


def rmsnorm_bf16(x: torch.Tensor, w: Optional[torch.Tensor], eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: f32 [T, n] -> bf16 [T, n] = w * x * rsqrt(mean(x^2) + eps); w=None converts only."""
    T, n = x.shape
    if out is None:
        out = torch.empty(T, n, dtype=torch.bfloat16, device=x.device)
    cl.check(cl.lib().dl_rmsnorm_bf16(x.data_ptr(), x.stride(0), w.data_ptr() if w is not None else None, out.data_ptr(), out.stride(0),
                                      n, eps, T, cl.stream_ptr()), "rmsnorm_bf16")
    return out


def gemv_q40_argmax_rows(w: DeviceQ40, x: torch.Tensor, *, norm_w: torch.Tensor, eps: float, out: torch.Tensor, arg_val: torch.Tensor,
                         arg_idx: torch.Tensor, arg_counter: torch.Tensor, tokens: torch.Tensor, vocab_limit: int = 0,
                         num_sms: int = 0) -> None:
    """Fused logits + per-row arg-max of nb = x.shape[0] (2, 4 or 8) rows on the TMA kernel (the verify step of speculative
    decoding): out [nb][d] = logits of rmsnorm(x[b]); tokens[b] = lowest-index maximum of row b among rows < vocab_limit (0: all).
    arg_val / arg_idx: nb x grid entries; arg_counter: zero, left at zero. Raises with code 1 where the shape does not fit."""
    if num_sms == 0:
        num_sms = torch.cuda.get_device_properties(x.device).multi_processor_count
    cl.check(cl.lib().dl_gemv_q40_argmax_rows(w.qs.data_ptr(), w.scales.data_ptr(), w.d, w.n, x.data_ptr(), norm_w.data_ptr(), eps,
                                              out.data_ptr(), arg_val.data_ptr(), arg_idx.data_ptr(), arg_counter.data_ptr(),
                                              tokens.data_ptr(), vocab_limit, x.shape[0], num_sms, cl.stream_ptr()), "gemv_q40_argmax_rows")
