"""ctypes binding of the sm_90a kernel/runtime library (csrc/cuda -> distributed_llama_b200/_cuda.so).

The library is torch-free: tensors cross the boundary as raw device pointers + the current CUDA stream handle.
If the library is missing on a machine with a GPU we build it; failures are loud (no eager fallback).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

from .. import _build

_lib: Optional[C.CDLL] = None

u32, u64, i32, f32, vp = C.c_uint32, C.c_uint64, C.c_int, C.c_float, C.c_void_p


class EngineConfig(C.Structure):
    _fields_ = [(n, u32) for n in ("dim", "nLayers", "nHeads", "nKvHeads", "headDim", "ffDim", "vocab", "seqLen",
                                   "nExperts", "nActiveExperts", "maxBatch", "nSplits", "rank", "nRanks", "numSms")] + \
               [("eps", f32), ("usePdl", u32), ("moeFirstExpert", u32), ("moeNumLocal", u32), ("wType", u32), ("hiddenAct", u32),
                                             ("kvType", u32), ("maxPrefill", u32)]


class LayerPtrs(C.Structure):
    _fields_ = [(n, vp) for n in ("qkvQs", "qkvSc", "woQs", "woSc", "w13Qs", "w13Sc", "w2Qs", "w2Sc",
                                  "norm0", "norm1", "qNorm", "kNorm", "moeGate", "kCache", "vCache", "kScale", "vScale")]


class GlobalPtrs(C.Structure):
    _fields_ = [("embedding", vp), ("embeddingPeers", vp * 8), ("embRowsPerRank", u32), ("finalNorm", vp), ("wclsQs", vp), ("wclsSc", vp), ("rope", vp), ("vocabFull", u32),
                ("tokens", vp), ("pos", vp), ("x", vp), ("logits", vp), ("history", vp)]


class CommPtrs(C.Structure):
    _fields_ = [("nRanks", u32), ("rank", u32), ("arena", vp * 8), ("mcArena", vp)]


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build_cuda()
    L = C.CDLL(str(path))
    sizes = (C.c_uint32 * 4)()
    L.dl_abi_struct_sizes(sizes)
    if [C.sizeof(s) for s in (EngineConfig, LayerPtrs, GlobalPtrs, CommPtrs)] != list(sizes):
        raise RuntimeError(f"{path}: sizes {list(sizes)} of EngineConfig, LayerPtrs, GlobalPtrs, CommPtrs differ from their ctypes mirrors")
    L.dl_repack_q40.argtypes = [vp, u64, u64, u32, u32, vp, vp, u32, u32, u32, vp]
    L.dl_repack_q40.restype = i32
    L.dl_dequant_device_q40.argtypes = [vp, vp, u32, u32, vp, vp]
    L.dl_dequant_device_q40.restype = i32
    L.dl_gemv_q40.argtypes = [i32, i32, i32, vp, vp, u32, u32, vp, u32, vp, f32, vp, u32, i32, vp, i32, i32, u32]
    L.dl_gemv_q40.restype = i32
    L.dl_gemv_q40_plan.argtypes = [i32, i32, i32, u32, u32, i32, i32, C.POINTER(C.c_int)]
    L.dl_gemv_q40_plan.restype = i32
    L.dl_gemv_q40_argmax.argtypes = [vp, vp, u32, u32, vp, vp, f32, vp, vp, vp, vp, vp, vp, vp, u32, u32, u32, i32, vp]
    L.dl_gemv_q40_argmax.restype = i32
    L.dl_argmax_advance.argtypes = [vp, u32, vp, vp, vp, u32, vp]
    L.dl_argmax_advance.restype = i32
    L.dl_gemv_dense.argtypes = [i32, i32, i32, i32, vp, u32, u32, vp, u32, vp, f32, vp, u32, i32, vp, i32, u32]
    L.dl_gemv_dense.restype = i32
    L.dl_gemv_dense_smem_bytes.argtypes = [u32, u32, i32, i32]
    L.dl_gemv_dense_smem_bytes.restype = u64
    L.dl_gemm_q40_tc.argtypes = [i32, vp, vp, u32, u32, vp, u32, u32, vp, u32, i32, u32, vp, i32, i32]
    L.dl_gemm_q40_tc.restype = i32
    L.dl_gemm_q40_tc_plan.argtypes = [i32, u32, u32, u32, u32, i32, i32, C.POINTER(C.c_int)]
    L.dl_gemm_q40_tc_plan.restype = i32
    L.dl_rmsnorm_bf16.argtypes = [vp, u32, vp, vp, u32, u32, f32, u32, vp]
    L.dl_rmsnorm_bf16.restype = i32
    L.dl_attn_prefill_tc.argtypes = [vp, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_attn_prefill_tc.restype = i32
    L.dl_rope_kv.argtypes = [vp, u32, vp, vp, vp, vp, f32, u32, u32, u32, u32, vp, vp, i32, vp]
    L.dl_rope_kv.restype = i32
    L.dl_rope_kv_q80.argtypes = [vp, u32, vp, vp, vp, vp, f32, u32, u32, u32, u32, vp, vp, vp, vp, i32, vp]
    L.dl_rope_kv_q80.restype = i32
    L.dl_attn_decode_q80.argtypes = [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp, i32, vp]
    L.dl_attn_decode_q80.restype = i32
    L.dl_attn_fused_q80.argtypes = [vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, vp]
    L.dl_attn_fused_q80.restype = i32
    L.dl_choice_attn_only_q80.argtypes = [vp, u32, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_choice_attn_only_q80.restype = i32
    L.dl_slot_attn_q80.argtypes = [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_slot_attn_q80.restype = i32
    L.dl_attn_prefill_tc_q80.argtypes = [vp, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, vp, vp, u32, vp]
    L.dl_attn_prefill_tc_q80.restype = i32
    L.dl_attn_decode.argtypes = [vp, u32, vp, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp, i32, vp]
    L.dl_attn_decode.restype = i32
    L.dl_attn_fused.argtypes = [vp, vp, vp, vp, vp, f32, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, vp]
    L.dl_attn_fused.restype = i32
    L.dl_moe_router.argtypes = [vp, vp, vp, f32, u32, u32, u32, vp, vp, vp, vp, i32, vp]
    L.dl_moe_router.restype = i32
    L.dl_gemm_q40_tc_grouped.argtypes = [i32, vp, vp, u32, u32, u32, vp, u32, u32, u32, vp, vp, vp, u32, i32, u32, vp]
    L.dl_gemm_q40_tc_grouped.restype = i32
    L.dl_moe_prefill_ffn.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, f32, i32, u32, vp, vp, vp]
    L.dl_moe_prefill_ffn.restype = i32
    L.dl_moe_decode_ffn.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, f32, vp, vp, vp, vp, vp, vp, vp, u32, u32, vp]
    L.dl_moe_decode_ffn.restype = i32
    L.dl_moe_decode_ffn_dense.argtypes = [i32, vp, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, f32, vp, vp, vp, vp, vp, vp, vp, u32, u32, vp]
    L.dl_moe_decode_ffn_dense.restype = i32
    L.dl_engine_create.argtypes = [C.POINTER(EngineConfig)]
    L.dl_engine_create.restype = vp
    L.dl_engine_destroy.argtypes = [vp]
    L.dl_engine_destroy.restype = None
    L.dl_engine_set_layer.argtypes = [vp, u32, C.POINTER(LayerPtrs)]
    L.dl_engine_set_layer.restype = i32
    L.dl_engine_set_globals.argtypes = [vp, C.POINTER(GlobalPtrs)]
    L.dl_engine_set_globals.restype = i32
    L.dl_engine_enable_mega.argtypes = [vp, i32]
    L.dl_engine_enable_mega.restype = i32
    L.dl_engine_set_vocab_limit.argtypes = [vp, u32]
    L.dl_engine_set_vocab_limit.restype = i32
    L.dl_engine_arena_bytes.argtypes = [vp]
    L.dl_engine_arena_bytes.restype = u64
    L.dl_engine_set_comm.argtypes = [vp, C.POINTER(CommPtrs)]
    L.dl_engine_set_comm.restype = i32
    for name, args in (("dl_comm_alloc", [C.c_size_t, C.POINTER(vp)]), ("dl_comm_free", [vp]), ("dl_comm_ipc_handle", [vp, vp]),
                       ("dl_comm_ipc_open", [vp, C.POINTER(vp)]), ("dl_comm_ipc_close", [vp]), ("dl_comm_memset", [vp, i32, C.c_size_t, vp])):
        getattr(L, name).argtypes = args
        getattr(L, name).restype = i32
    L.dl_vmm_supported.argtypes = [C.POINTER(C.c_int)]
    L.dl_vmm_supported.restype = i32
    L.dl_vmm_create.argtypes = [u32, u32, C.c_size_t, C.c_char_p, i32]
    L.dl_vmm_create.restype = vp
    L.dl_vmm_connect.argtypes = [vp]
    L.dl_vmm_connect.restype = i32
    L.dl_vmm_ptr.argtypes = [vp, u32]
    L.dl_vmm_ptr.restype = vp
    L.dl_vmm_mc_ptr.argtypes = [vp]
    L.dl_vmm_mc_ptr.restype = vp
    L.dl_vmm_bytes.argtypes = [vp]
    L.dl_vmm_bytes.restype = C.c_size_t
    L.dl_vmm_destroy.argtypes = [vp]
    L.dl_vmm_destroy.restype = None
    L.dl_vmm_selftest_kernel.argtypes = [vp, u32, i32, vp]
    L.dl_vmm_selftest_kernel.restype = i32
    L.dl_engine_set_trace.argtypes = [vp, vp, u32]
    L.dl_engine_set_trace.restype = i32
    L.dl_engine_sampler_seed.argtypes = [vp, C.c_uint64]
    L.dl_engine_sampler_seed.restype = i32
    L.dl_engine_sample.argtypes = [vp, f32, f32, vp]
    L.dl_engine_sample.restype = i32
    L.dl_sample_logits.argtypes = [vp, vp, u32, f32, f32, vp, vp, vp]
    L.dl_sample_logits.restype = i32
    L.dl_sample_rows.argtypes = [vp, u32, vp, u32, f32, f32, vp, vp, u32, u32, vp]
    L.dl_sample_rows.restype = i32
    L.dl_sample_rows_controlled.argtypes = [vp, u32, vp, u32, f32, f32, vp, vp, u32, u32, vp, vp, u32, f32, f32, vp]
    L.dl_sample_rows_controlled.restype = i32
    L.dl_engine_set_sampling_controls.argtypes = [vp, f32, f32, C.POINTER(C.c_int32), C.POINTER(f32), i32, u32, vp]
    L.dl_engine_set_sampling_controls.restype = i32
    L.dl_engine_set_sampling_filters.argtypes = [vp, u32, f32]
    L.dl_engine_set_sampling_filters.restype = i32
    L.dl_sample_logits_filtered.argtypes = [vp, vp, u32, f32, f32, u32, f32, vp, vp, vp]
    L.dl_sample_logits_filtered.restype = i32
    L.dl_sample_rows_filtered.argtypes = [vp, u32, vp, u32, vp, vp, vp, vp, u32, u32, vp, u32, vp, u32, vp]
    L.dl_sample_rows_filtered.restype = i32
    L.dl_choice_attn.argtypes = [vp, u32, vp, vp, vp, vp, f32, vp, vp, u32, u32, u32, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_choice_attn.restype = i32
    L.dl_choice_attn_only.argtypes = [vp, u32, vp, vp, u32, u32, u32, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_choice_attn_only.restype = i32
    L.dl_engine_sampler_state.argtypes = [vp]
    L.dl_engine_sampler_state.restype = C.c_uint64
    L.dl_engine_sampler_seed_rows.argtypes = [vp, C.POINTER(C.c_uint64), i32]
    L.dl_engine_sampler_seed_rows.restype = i32
    L.dl_engine_sample_rows.argtypes = [vp, i32, u32, f32, f32, i32, vp]
    L.dl_engine_sample_rows.restype = i32
    L.dl_engine_choices_forward.argtypes = [vp, i32, u32, u32, u32, u32, vp]
    L.dl_engine_choices_forward.restype = i32
    L.dl_sample_rows_per_row.argtypes = [vp, u32, vp, u32, vp, vp, vp, u32, u32, vp, u32, vp, u32, vp]
    L.dl_sample_rows_per_row.restype = i32
    L.dl_slot_attn.argtypes = [vp, u32, vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_slot_attn.restype = i32
    ip = C.POINTER(C.c_int32)
    L.dl_engine_set_slots.argtypes = [vp, u32]
    L.dl_engine_set_slots.restype = i32
    L.dl_engine_slot_len.argtypes = [vp]
    L.dl_engine_slot_len.restype = u32
    L.dl_engine_set_slot_cache.argtypes = [vp, i32]
    L.dl_engine_set_slot_cache.restype = i32
    L.dl_engine_slot_reserve.argtypes = [vp, u32, u32]
    L.dl_engine_slot_reserve.restype = i32
    L.dl_engine_slot_trim.argtypes = [vp, u32, u32]
    L.dl_engine_slot_trim.restype = i32
    L.dl_engine_slot_release.argtypes = [vp, u32]
    L.dl_engine_slot_release.restype = i32
    L.dl_engine_free_pages.argtypes = [vp]
    L.dl_engine_free_pages.restype = u32
    L.dl_engine_slot_pages.argtypes = [vp, u32, ip, u32]
    L.dl_engine_slot_pages.restype = i32
    L.dl_slot_attn_paged.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.dl_slot_attn_paged.restype = i32
    L.dl_attn_prefill_tc_paged.argtypes = [vp, u32, u32, u32, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp, u32, vp]
    L.dl_attn_prefill_tc_paged.restype = i32
    L.dl_engine_slot_copy.argtypes = [vp, u32, u32, u32, vp]
    L.dl_engine_slot_copy.restype = i32
    L.dl_engine_slot_sampling.argtypes = [vp, u32, C.c_uint64, f32, f32, f32, f32, ip, C.POINTER(f32), i32, vp]
    L.dl_engine_slot_sampling.restype = i32
    L.dl_engine_slot_filters.argtypes = [vp, u32, u32, f32]
    L.dl_engine_slot_filters.restype = i32
    L.dl_engine_slots_forward.argtypes = [vp, ip, ip, u32, vp]
    L.dl_engine_slots_forward.restype = i32
    L.dl_engine_slots_step.argtypes = [vp, ip, ip, u32, ip, vp]
    L.dl_engine_slots_step.restype = i32
    L.dl_engine_slot_logprobs.argtypes = [vp, u32, i32]
    L.dl_engine_slot_logprobs.restype = i32
    L.dl_engine_slots_step_logprobs.argtypes = [vp, ip, ip, u32, ip, ip, vp]
    L.dl_engine_slots_step_logprobs.restype = i32
    L.dl_engine_logprobs.argtypes = [vp, i32, u32, ip, i32, i32, vp, vp]
    L.dl_engine_logprobs.restype = i32
    L.dl_logprobs_rows.argtypes = [vp, u32, u32, u32, u32, ip, vp, vp, u32, vp, u32, f32, f32, vp, vp, vp]
    L.dl_logprobs_rows.restype = i32
    L.dl_engine_sync_ns.argtypes = [vp]
    L.dl_engine_sync_ns.restype = C.c_uint64
    L.dl_engine_mega_active.argtypes = [vp]
    L.dl_engine_mega_active.restype = i32
    L.dl_engine_mega_copy_vectors.argtypes = [vp, vp, vp, vp, vp, vp]
    L.dl_engine_mega_copy_vectors.restype = i32
    L.dl_engine_aborted.argtypes = [vp]
    L.dl_engine_aborted.restype = i32
    L.dl_engine_set_trace_all.argtypes = [vp, i32]
    L.dl_engine_set_trace_all.restype = i32
    L.dl_engine_num_sms.argtypes = [vp]
    L.dl_engine_num_sms.restype = u32
    L.dl_engine_forward.argtypes = [vp, i32, i32, i32, vp]
    L.dl_engine_forward.restype = i32
    L.dl_engine_forward_part.argtypes = [vp, i32, u32, i32, vp, vp]
    L.dl_engine_forward_part.restype = i32
    L.dl_engine_prefill.argtypes = [vp, ip, u32, u32, i32, i32, vp]
    L.dl_engine_prefill.restype = i32
    up = C.POINTER(C.c_uint32)
    L.dl_engine_prefill_plan.argtypes = [vp, u32, u32, i32, up, u32]
    L.dl_engine_prefill_plan.restype = i32
    L.dl_prefill_plan.argtypes = [u32, u32, i32, u32, u32, u32, u32, u32, i32, up, u32]
    L.dl_prefill_plan.restype = i32
    L.dl_engine_prefill_scratch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dl_engine_prefill_scratch.restype = i32
    L.dl_engine_moe_scratch.argtypes = [vp, u32, i32, vp, vp, vp, vp, vp]
    L.dl_engine_moe_scratch.restype = i32
    L.dl_moe_scratch_caps.argtypes = [vp]
    L.dl_moe_scratch_caps.restype = None
    L.dl_engine_set_prefill_min_tc.argtypes = [vp, u32]
    L.dl_engine_set_prefill_min_tc.restype = i32
    L.dl_engine_decode_graph.argtypes = [vp, i32, vp]
    L.dl_engine_decode_graph.restype = i32
    L.dl_engine_graph_captured.argtypes = [vp]
    L.dl_engine_graph_captured.restype = i32
    L.dl_spec_round.argtypes = [vp, vp, i32, i32, i32, i32, ip, vp]
    L.dl_spec_round.restype = i32
    L.dl_engine_verify.argtypes = [vp, i32, ip, vp]
    L.dl_engine_verify.restype = i32
    L.dl_spec_accept.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, u32, u32, vp, vp]
    L.dl_spec_accept.restype = i32
    L.dl_gemv_q40_argmax_rows.argtypes = [vp, vp, u32, u32, vp, vp, f32, vp, vp, vp, vp, vp, u32, i32, i32, vp]
    L.dl_gemv_q40_argmax_rows.restype = i32
    L.dl_argmax_rows.argtypes = [vp, u32, u32, i32, vp, vp]
    L.dl_argmax_rows.restype = i32
    if L.dl_spec_result_words() != SPEC_RESULT_WORDS:
        raise RuntimeError(f"{path}: speculative result block of {L.dl_spec_result_words()} words, expected {SPEC_RESULT_WORDS}")
    _lib = L
    return L


_ERRORS = {
    -12: "prompt chunk larger than the prefill all-reduce slots of the peer arena",
    -30: "tensor-parallel slice too narrow for the fused all-reduce GEMV: the per-rank K of WO / W2 (heads/N * headDim, ffDim/N) "
         "must be a multiple of 128 — use fewer ranks, or DL_COLLECTIVES=nccl",
    -31: "mixture-of-experts up-projection shape not covered by the TMA GEMV",
    -32: "mixture-of-experts down-projection shape not covered by the TMA GEMV (per-rank expert ffDim must be a multiple of 128: use moe_mode=ep)",
    -33: "arg-max under tensor parallelism needs the fused logits kernel",
    -36: "mixture-of-experts prefill shape not covered (dim, ffDim multiples of 256, chunk <= 256 tokens)",
    -40: "the dense-weight GEMV has no in-kernel all-reduce (dense weight files use library collectives under tensor parallelism)",
    -41: "expert-routed dense-weight GEMV needs one token, the routing slots' expert indices and k >= 1",
    -53: "logit_bias token id outside the sampled vocabulary",
    -66: "a slot position past the rows the slot holds",
    -68: "the KV-cache page pool has too few free pages",
    -69: "paged KV-cache slots need the tensor-core prefill attention",
    -71: "speculative round at a position past the context",
    -72: "the draft model must be a second engine with the target's vocabulary and KV-cache float type",
    -73: "speculative decoding needs one GPU, dense q40 models and no KV-cache slots",
    -74: "device-side wait timed out during a speculative round",
    -75: "--draft-tokens must be 1, 3 or 7",
    -77: "out of device or pinned memory for the speculative-decoding state",
}

# Speculative rounds (dl_spec_round): int32 result block [accepted, emitted, drafts, position of the last emitted token, tokens...]
SPEC_RESULT_WORDS, SPEC_RESULT_HEAD = 12, 4

POOL_SHORT = -68   # dl_engine_slot_reserve / dl_engine_slot_copy: too few free pages, nothing changed
PAGE_ROWS = 64     # rows of a KV-cache page (paged slots)
SLOT_CACHE_LAYOUTS = ("split", "paged")   # --parallel-cache


def check(code: int, what: str) -> None:
    if code != 0:
        raise RuntimeError(f"{what} failed with code {code}" + (f": {_ERRORS[code]}" if code in _ERRORS else ""))


def stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


# KV-cache storage (EngineConfig.kvType): name of --kv-cache-float-type -> code
KV_CACHE_TYPES = {"bf16": 0, "q80": 1}

# Log-probabilities (csrc/cuda/logprobs.cu): int32 words of one row's result block, the largest top_logprobs, dl_engine_logprobs flags
LOGPROBS_WORDS, LOGPROBS_MAX_TOP = 44, 20
LP_CONTROLLED, LP_SHARED_ROW = 1, 2


def decode_logprobs(words) -> tuple:
    """One row's result block (LOGPROBS_WORDS int32 values) -> (chosen id, its logprob, [(id, logprob), ...] top entries)."""
    import struct
    w = [int(x) for x in words]
    f = lambda bits: struct.unpack("<f", struct.pack("<i", bits))[0]
    k = w[2]
    return w[0], f(w[1]), [(w[4 + 2 * j], f(w[5 + 2 * j])) for j in range(k)]

PRO_RMSNORM, PRO_PLAIN = 0, 1
EPI_STORE, EPI_RESIDUAL, EPI_SWIGLU, EPI_ARGMAX = 0, 1, 2, 3
GEPI_STORE_F32, GEPI_RESIDUAL, GEPI_SWIGLU_BF16 = 0, 1, 2
