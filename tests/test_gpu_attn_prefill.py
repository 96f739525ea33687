"""Tensor-core prompt-chunk attention (csrc/cuda/attn_prefill_tc.cu) vs a plain PyTorch f32 reference of the same op:
causal softmax(q.k^T / sqrt(hd)).v over a bf16 head-major KV cache, GQA, chunk of T tokens starting at position p0."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _reference(q, k_cache, v_cache, p0, n_heads, n_kv, hd):
    T = q.shape[0]
    kv_mul = n_heads // n_kv
    out = torch.zeros(T, n_heads * hd, device=q.device)
    for h in range(n_heads):
        g = h // kv_mul
        qh = q[:, h * hd:(h + 1) * hd]                       # [T, hd]
        kk = k_cache[g, :p0 + T].float()                     # [P, hd]
        vv = v_cache[g, :p0 + T].float()
        s = qh @ kk.T / math.sqrt(hd)                        # [T, P]
        pos = torch.arange(p0 + T, device=q.device)[None, :]
        row = (p0 + torch.arange(T, device=q.device))[:, None]
        s = s.masked_fill(pos > row, float("-inf"))
        out[:, h * hd:(h + 1) * hd] = torch.softmax(s, dim=-1) @ vv
    return out


@pytest.mark.parametrize("n_heads,n_kv,hd", [(32, 8, 128), (8, 8, 128), (40, 8, 128), (32, 4, 128), (32, 8, 64), (4, 1, 128), (6, 2, 64)])
@pytest.mark.parametrize("T,p0", [(64, 0), (5, 0), (33, 100), (200, 0), (192, 300), (1, 7)])
def test_attn_prefill_tc_matches_reference(n_heads, n_kv, hd, T, p0):
    from distributed_llama_b200.ops import cuda_lib as cl
    lib = cl.lib()
    torch.manual_seed(n_heads * 1000 + T + p0)
    seq = 640
    q_dim, kv_dim = n_heads * hd, n_kv * hd
    stride = q_dim + 2 * kv_dim
    qkv = torch.randn(T, stride, device="cuda")
    k_cache = (torch.randn(n_kv, seq, hd, device="cuda") * 0.7).bfloat16()
    v_cache = torch.randn(n_kv, seq, hd, device="cuda").bfloat16()
    out = torch.full((T, q_dim), float("nan"), device="cuda", dtype=torch.bfloat16)
    rc = lib.dl_attn_prefill_tc(qkv.data_ptr(), stride, T, p0, n_heads, n_kv, hd, seq, k_cache.data_ptr(), v_cache.data_ptr(),
                                out.data_ptr(), q_dim, cl.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    ref = _reference(qkv[:, :q_dim], k_cache, v_cache, p0, n_heads, n_kv, hd)
    got = out.float()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    assert err < 0.03 * ref.abs().max().item() + 2e-3, (err, ref.abs().max().item())
