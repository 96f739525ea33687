"""Tensor-core prefill GEMM (q40 dequant fused into the prologue) vs a plain PyTorch f32 reference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_kernels import _rand_q40, _device_q40   # noqa: E402


@pytest.mark.parametrize("variant", ["ldg", "tma"])
@pytest.mark.parametrize("d,n,T", [(256, 256, 16), (128, 64, 1), (384, 512, 17), (6144, 4096, 64), (4096, 14336, 64),
                                   (1024, 1792, 200), (2048, 4096, 256), (1000, 2176, 33), (28672, 4096, 100), (4096, 4096, 192),
                                   (4096, 14336, 128)])
def test_gemm_store_f32(d, n, T, variant):
    if variant == "tma" and n % 256:
        pytest.skip("TMA-staged variant needs n % 256 == 0")
    from distributed_llama_b200 import ops
    raw, wq = _rand_q40(d, n, seed=5)
    w = _device_q40(raw, d, n)
    torch.manual_seed(2)
    act = torch.randn(T, n, device="cuda").bfloat16()
    out = torch.full((T, d), float("nan"), device="cuda")
    ops.gemm_q40_tc(w, act, epi=ops.GEPI_STORE_F32, out=out, variant=variant)
    torch.cuda.synchronize()
    ref = act.float() @ torch.from_numpy(wq).cuda().T
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err < 0.02 * scale + 1e-3, (err, scale)


@pytest.mark.parametrize("cluster", ["1", "0"])
def test_gemm_split_k_over_token_tiles(cluster, monkeypatch):
    """Llama-3.1-8B w2 at a 128-token chunk: split-K over 2 token tiles, reduced inside a thread-block cluster or (cluster = 0)
    through the global scratch; residual epilogue."""
    from distributed_llama_b200 import ops
    monkeypatch.setenv("DL_GEMM_CLUSTER", cluster)
    d, n, T = 4096, 14336, 128
    raw, wq = _rand_q40(d, n, seed=8)
    w = _device_q40(raw, d, n)
    torch.manual_seed(4)
    act = torch.randn(T, n, device="cuda").bfloat16()
    x = torch.randn(T, d, device="cuda")
    ref = x + act.float() @ torch.from_numpy(wq).cuda().T
    ops.gemm_q40_tc(w, act, epi=ops.GEPI_RESIDUAL, out=x, variant="tma")
    torch.cuda.synchronize()
    assert (x - ref).abs().max().item() < 0.02 * ref.abs().max().item() + 1e-3


def test_gemm_residual_and_swiglu():
    from distributed_llama_b200 import ops
    d, n, T = 1024, 1024, 48
    raw, wq = _rand_q40(d, n, seed=6)
    w = _device_q40(raw, d, n)
    wt = torch.from_numpy(wq).cuda()
    torch.manual_seed(3)
    act = torch.randn(T, n, device="cuda").bfloat16()
    x = torch.randn(T, d, device="cuda")
    x0 = x.clone()
    ops.gemm_q40_tc(w, act, epi=ops.GEPI_RESIDUAL, out=x)
    ref = x0 + act.float() @ wt.T
    assert (x - ref).abs().max().item() < 0.03 * ref.abs().max().item()
    h = torch.zeros(T, d // 2, device="cuda", dtype=torch.bfloat16)
    ops.gemm_q40_tc(w, act, epi=ops.GEPI_SWIGLU_BF16, out=h)
    full = act.float() @ wt.T
    refh = torch.nn.functional.silu(full[:, 0::2]) * full[:, 1::2]
    assert (h.float() - refh).abs().max().item() < 0.03 * refh.abs().max().item() + 0.02


def test_rmsnorm_bf16():
    from distributed_llama_b200 import ops
    x = torch.randn(37, 4096, device="cuda") * 3
    w = 1 + 0.1 * torch.randn(4096, device="cuda")
    y = ops.rmsnorm_bf16(x, w, 1e-5)
    ref = w * x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5)
    assert (y.float() - ref).abs().max().item() < 0.03
