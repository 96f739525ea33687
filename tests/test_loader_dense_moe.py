"""Qwen3-MoE files with f32 / f16 / q80 weights: the loader's expert layout and its tensor- and expert-parallel slices (CPU only).

The device layout is w13 [nLocal][2 * ff][dim] (gate and up rows of an expert interleaved) and w2 [nLocal][dim][ff]. Under "tp"
every rank holds every expert's ff slice; under "ep" it holds nExperts / nRanks whole experts."""
import numpy as np
import pytest
import torch

WTYPES = ("f32", "f16", "q80")


@pytest.fixture(scope="module")
def moe_files(tmp_path_factory):
    from distributed_llama_b200.formats import quants
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model
    root = tmp_path_factory.mktemp("dense_moe")
    out = {}
    for wt in WTYPES:
        path = str(root / f"tiny-qwen3-moe-{wt}.m")
        write_synthetic_model(path, get_config("tiny-qwen3-moe"), weights_float_type=quants.parse_float_type(wt), seed=7)
        out[wt] = path
    return out


def _experts(W, which):
    """[nLocal][rows][cols] view of a layer-0 expert matrix of DeviceWeights W."""
    L = W.layers[0]
    h = W.header
    if which == "w13":
        return L.w13.data.view(W.n_local_experts, 2 * W.ff_dim, h.dim)
    return L.w2.data.view(W.n_local_experts, h.dim, W.ff_dim)


@pytest.mark.parametrize("wt", WTYPES)
@pytest.mark.parametrize("n_ranks", [2, 4])
@pytest.mark.parametrize("mode", ["tp", "ep"])
def test_expert_slices_reassemble(moe_files, wt, n_ranks, mode):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    mf = ModelFile(moe_files[wt])
    h = mf.header
    full = load_device_weights(mf, 0, 1, device="cpu")
    parts = [load_device_weights(mf, r, n_ranks, device="cpu", moe_mode=mode) for r in range(n_ranks)]
    assert full.weight_kind == (2 if wt == "f16" else 1)
    assert full.n_local_experts == h.n_experts and full.first_expert == 0
    dt = torch.float16 if wt == "f16" else torch.float32
    for l in range(h.n_layers):
        F = full.layers[l]
        assert F.w13.data.dtype == dt and F.w2.data.dtype == dt
        assert F.moe_gate.dtype == torch.float32 and tuple(F.moe_gate.shape) == (h.n_experts, h.dim)
        assert all(torch.equal(p.layers[l].moe_gate, F.moe_gate) for p in parts)
        for e in range(h.n_experts):   # the full layout against the file, expert by expert
            w1, w2, w3 = (torch.from_numpy(mf.tensor_f32(mf.entry(n, l, e))).to(dt)
                          for n in ("block_matmul_w1", "block_matmul_w2", "block_matmul_w3"))
            f13 = F.w13.data.view(h.n_experts, 2 * h.ff_dim, h.dim)[e]
            assert torch.equal(f13[0::2], w1) and torch.equal(f13[1::2], w3)
            assert torch.equal(F.w2.data.view(h.n_experts, h.dim, h.ff_dim)[e], w2)
    for which in ("w13", "w2"):
        fx = _experts(full, which)
        px = [_experts(p, which) for p in parts]
        if mode == "ep":
            assert [p.moe_mode for p in parts] == ["ep"] * n_ranks
            assert [p.first_expert for p in parts] == [r * h.n_experts // n_ranks for r in range(n_ranks)]
            assert all(p.n_local_experts == h.n_experts // n_ranks and p.ff_dim == h.ff_dim for p in parts)
            assert torch.equal(torch.cat(px, 0), fx)
        else:
            assert all(p.moe_mode == "tp" and p.n_local_experts == h.n_experts and p.ff_dim == h.ff_dim // n_ranks for p in parts)
            if which == "w2":
                assert torch.equal(torch.cat(px, 2), fx)
            else:
                for k in (0, 1):   # gate rows / up rows
                    assert torch.equal(torch.cat([x[:, k::2] for x in px], 1), fx[:, k::2])


def test_auto_mode_picks_ep_for_narrow_slices(moe_files):
    """`auto` is the q40 loader's rule: expert parallelism when a rank's ff slice would not be a multiple of 128 columns."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    mf = ModelFile(moe_files["f16"])
    assert mf.header.ff_dim == 256
    assert load_device_weights(mf, 0, 2, device="cpu").moe_mode == "tp"
    assert load_device_weights(mf, 1, 4, device="cpu").moe_mode == "ep"


def test_q80_experts_are_exact(moe_files):
    """q80 expert blocks become int8 x f16 scale in f32, computed here straight from the file's bytes."""
    from distributed_llama_b200.formats import ModelFile, quants
    from distributed_llama_b200.models.loader import load_device_weights
    mf = ModelFile(moe_files["q80"])
    h = mf.header
    W = load_device_weights(mf, 0, 1, device="cpu")

    def exact(entry):
        b = np.asarray(mf.raw(entry)).reshape(-1, quants.Q80_BYTES)
        scale = b[:, :2].copy().view(np.float16).astype(np.float32)
        q = b[:, 2:].copy().view(np.int8).astype(np.float32)
        return torch.from_numpy((q * scale).reshape(entry.d, entry.n))

    for l in range(h.n_layers):
        w13 = W.layers[l].w13.data.view(h.n_experts, 2 * h.ff_dim, h.dim)
        w2 = W.layers[l].w2.data.view(h.n_experts, h.dim, h.ff_dim)
        for e in range(h.n_experts):
            assert torch.equal(w13[e, 0::2], exact(mf.entry("block_matmul_w1", l, e)))
            assert torch.equal(w13[e, 1::2], exact(mf.entry("block_matmul_w3", l, e)))
            assert torch.equal(w2[e], exact(mf.entry("block_matmul_w2", l, e)))


def _device_layout_forward(mf, parts, tokens):
    """PyTorch emulation of the engine on the device layout: q|k|v concatenated, adjacent rotary pairs, f32 router -> softmax ->
    top-k (renormalised) -> per-expert interleaved W1|W3 SwiGLU -> W2, weighted and summed in routing-slot order; every rank's
    partial sums (its heads, its expert slices or whole experts) added as the all-reduce would."""
    h = mf.header
    hd, eps = h.head_dim, h.norm_epsilon
    caches = [[([], []) for _ in range(h.n_layers)] for _ in parts]

    def rms(v, w):
        return w * v * torch.rsqrt((v * v).mean(-1, keepdim=True) + eps)

    def rope(v, pos, table):
        cs = table[pos]
        a, b = v[:, 0::2], v[:, 1::2]
        out = torch.empty_like(v)
        out[:, 0::2] = a * cs[:, 0] - b * cs[:, 1]
        out[:, 1::2] = a * cs[:, 1] + b * cs[:, 0]
        return out

    rows = []
    for pos, tok in enumerate(tokens):
        x = parts[0].embedding[tok].float().clone()
        for l in range(h.n_layers):
            partial = torch.zeros_like(x)
            for r, W in enumerate(parts):
                L = W.layers[l]
                nh, nkv = W.n_heads, W.n_kv_heads
                qkv = L.qkv.data.float() @ rms(x, L.norm0)
                q = rms(qkv[: nh * hd].view(nh, hd), L.q_norm)
                k = rms(qkv[nh * hd: (nh + nkv) * hd].view(nkv, hd), L.k_norm)
                v = qkv[(nh + nkv) * hd:].view(nkv, hd)
                q, k = rope(q, pos, W.rope), rope(k, pos, W.rope)
                kc, vc = caches[r][l]
                kc.append(k); vc.append(v)
                K, V = torch.stack(kc, 1), torch.stack(vc, 1)
                z = [torch.softmax((K[i // (nh // nkv)] @ q[i]) / hd ** 0.5, -1) @ V[i // (nh // nkv)] for i in range(nh)]
                partial += L.wo.data.float() @ torch.cat(z)
            x = x + partial
            xn = rms(x, parts[0].layers[l].norm1)
            probs = torch.softmax(parts[0].layers[l].moe_gate @ xn, -1)
            topv, topi = torch.topk(probs, h.n_active_experts)
            topv = topv / topv.sum()
            partial = torch.zeros_like(x)
            for W in parts:
                w13, w2 = _experts_layer(W, l)
                for s in range(h.n_active_experts):
                    e = int(topi[s]) - W.first_expert
                    if 0 <= e < W.n_local_experts:
                        gu = w13[e].float() @ xn
                        partial += topv[s] * (w2[e].float() @ (torch.nn.functional.silu(gu[0::2]) * gu[1::2]))
            x = x + partial
        xn = rms(x, parts[0].final_norm)
        rows.append(torch.cat([W.wcls.data.float() @ xn for W in parts]))
    return torch.stack(rows)


def _experts_layer(W, l):
    L, h = W.layers[l], W.header
    return (L.w13.data.view(W.n_local_experts, 2 * W.ff_dim, h.dim), L.w2.data.view(W.n_local_experts, h.dim, W.ff_dim))


@pytest.mark.parametrize("wt,n_ranks,mode", [("f32", 1, "tp"), ("f16", 2, "tp"), ("q80", 2, "ep"), ("f32", 4, "ep"), ("f16", 4, "tp")])
def test_device_layout_forward_matches_oracle(moe_files, wt, n_ranks, mode):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    mf = ModelFile(moe_files[wt])
    parts = [load_device_weights(mf, r, n_ranks, device="cpu", moe_mode=mode) for r in range(n_ranks)]
    toks = [3, 17, 250, 9, 44, 101]
    got = _device_layout_forward(mf, parts, toks)
    ref = OracleModel(mf, act_quant="none").forward(toks, 0)
    assert (got - ref).abs().max().item() < 2e-3
