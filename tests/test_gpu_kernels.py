"""Device q40 repack (csrc/cuda/repack.cu) against the CPU dequantisation of the same blocks. The decode GEMVs are tested in
tests/test_gpu_gemv.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rand_q40(d, n, seed=0, std=None):
    from distributed_llama_b200.formats import quants
    rng = np.random.default_rng(seed)
    w = rng.standard_normal((d, n)).astype(np.float32) * (std or 1.0 / np.sqrt(n))
    raw = quants.quantize_q40(w)                         # [d*n/32, 18]
    wq = quants.dequantize_q40(raw).reshape(d, n)        # what the file really stores
    return raw.reshape(-1), wq


def _device_q40(raw, d, n, **kw):
    from distributed_llama_b200.ops import DeviceQ40, repack_q40
    dst = DeviceQ40.empty(d, n)
    repack_q40(torch.from_numpy(raw).cuda(), d, n, dst, **kw)
    return dst


def test_repack_roundtrip():
    d, n = 96, 256
    raw, wq = _rand_q40(d, n)
    dq = _device_q40(raw, d, n)
    torch.testing.assert_close(dq.to_f32().cpu(), torch.from_numpy(wq), rtol=0, atol=0)


def test_repack_column_slice_and_interleave():
    from distributed_llama_b200.ops import DeviceQ40, repack_q40
    d, n = 64, 512
    raw, wq = _rand_q40(d, n, seed=1)
    # column slice [128, 384)
    dst = DeviceQ40.empty(d, 256)
    repack_q40(torch.from_numpy(raw).cuda(), d, 256, dst, src_row_pitch=n // 32 * 18, src_col_byte_offset=128 // 32 * 18)
    torch.testing.assert_close(dst.to_f32().cpu(), torch.from_numpy(wq[:, 128:384].copy()), rtol=0, atol=0)
    # row interleave (w1/w3)
    raw2, wq2 = _rand_q40(d, n, seed=2)
    both = DeviceQ40.empty(2 * d, n)
    repack_q40(torch.from_numpy(raw).cuda(), d, n, both, dst_row_stride=2, dst_row_offset=0)
    repack_q40(torch.from_numpy(raw2).cuda(), d, n, both, dst_row_stride=2, dst_row_offset=1)
    full = both.to_f32().cpu().numpy()
    np.testing.assert_array_equal(full[0::2], wq)
    np.testing.assert_array_equal(full[1::2], wq2)
    # NeoX -> interleaved head re-ordering
    hd = 32
    perm = DeviceQ40.empty(d, n)
    repack_q40(torch.from_numpy(raw).cuda(), d, n, perm, head_dim=hd)
    got = perm.to_f32().cpu().numpy().reshape(d // hd, hd, n)
    ref = wq.reshape(d // hd, hd, n)
    np.testing.assert_array_equal(got[:, 0::2], ref[:, : hd // 2])
    np.testing.assert_array_equal(got[:, 1::2], ref[:, hd // 2:])
