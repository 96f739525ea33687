"""Mixture-of-experts decode with dense (f32 / f16) expert matrices: the expert-routed mode of the dense GEMV (gemv_dense.cu)
through `dl_moe_decode_ffn_dense`, the engine on Qwen3-MoE f32 / f16 / q80 files, and the front ends.

Kernel references are float64 over exactly the values the kernel multiplies: the exact expert weights (f16 values are exact in
f32 / float64), the float64 rmsnorm of x for W1|W3, and the kernel's own h for W2. They take the routing the kernel used (ids and
weights read back), so a near-tie in the f32 router cannot fail them; the chosen set is checked against float64 separately
wherever the k-th and (k+1)-th router logits are clearly apart.

Bounds (S = sum |a * w| over the dot product of an output, u = 2^-24):
* f32 dot product: a lane accumulates at most n / 32 products with fmaf (n <= 2048: 64), then a 5-step warp tree adds the lanes.
  Along any path that is at most 69 roundings, each at most u times a partial sum no larger than S: |err| <= 69 u S < 2^-17 S.
* Activations of W1|W3: rsqrtf, the f32 sum of squares and the products round the normalised vector to within 2^-18 relative of
  float64, which adds 2^-18 S.
* SwiGLU h = silu(g) * up with __expf and fast division: 2^-19 relative; the errors of g and up carry through |silu'| <= 1.1.
* The combine: weight * product, the sum of k slots and the add into `out`: k + 2 roundings of at most u of the magnitudes added.
At 2048 / 768 / 128 / 8 these bounds are about 1e-4 of max|Δx|, far below the 2e-2 the dense engine tests allow.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-6
SILU = 0
SHAPE_30B = (2048, 768, 128, 8)
SHAPE_TINY = (256, 256, 8, 2)
C_DOT = 2.0 ** -17
REL_NORM = 2.0 ** -18
REL_SILU = 2.0 ** -19


def _cl():
    from distributed_llama_b200.ops import cuda_lib as cl
    return cl


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def expert_weights(dim, ff, E, dtype, seed=5):
    """w13 [E][2ff][dim] (gate / up rows interleaved), w2 [E][dim][ff], in the weight type under test."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    w13 = (torch.randn(E, 2 * ff, dim, device="cuda", generator=g) * dim ** -0.5).to(dtype)
    w2 = (torch.randn(E, dim, ff, device="cuda", generator=g) * (0.5 * ff ** -0.5)).to(dtype)
    return w13, w2


def inputs(dim, E, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    x = torch.randn(dim, device="cuda", generator=g)
    norm = 1.0 + 0.1 * torch.randn(dim, device="cuda", generator=g)
    gate = torch.randn(E, dim, device="cuda", generator=g) * dim ** -0.5
    return x, norm, gate


class Bufs:
    def __init__(self, dim, ff, E, k, num_sms):
        z = dict(device="cuda")
        self.logits = torch.full((E,), float("nan"), **z)
        self.counter = torch.zeros(1 + 16, dtype=torch.int32, **z)
        self.ids = torch.full((k,), -1, dtype=torch.int32, **z)
        self.wts = torch.full((k,), float("nan"), **z)
        self.h = torch.full((k, ff), float("nan"), **z)
        self.scratch = torch.full((k, dim), float("nan"), **z)
        self.n_ctr = max(1, num_sms // k)
        self.counters = torch.zeros(self.n_ctr + 16, dtype=torch.int32, **z)
        self.counters[self.n_ctr:] = 0x7eadbeef
        self.counter[1:] = 0x7eadbeef

    def check(self, what):
        assert (self.counter[:1] == 0).all() and (self.counter[1:] == 0x7eadbeef).all(), f"{what}: router counter"
        assert (self.counters[:self.n_ctr] == 0).all(), f"{what}: slot counters not reset"
        assert (self.counters[self.n_ctr:] == 0x7eadbeef).all(), f"{what}: slot counters written past their end"


def ffn_call(wtype, x, out0, norm, gate, w13, w2, ff, k, num_sms, bufs, first=0, n_local=None):
    """One token; returns (out0 + weighted expert sum, h [k][ff], ids, weights). w13 / w2 hold experts [first, +n_local)."""
    cl = _cl()
    dim, E = x.shape[0], gate.shape[0]
    n_local = E - first if n_local is None else n_local
    w13l, w2l = w13[first:first + n_local].contiguous(), w2[first:first + n_local].contiguous()
    out = out0.clone()
    cl.check(cl.lib().dl_moe_decode_ffn_dense(wtype, x.data_ptr(), out.data_ptr(), norm.data_ptr(), gate.data_ptr(), w13l.data_ptr(),
                                              w2l.data_ptr(), dim, ff, E, k, first, n_local, EPS, bufs.logits.data_ptr(),
                                              bufs.counter.data_ptr(), bufs.ids.data_ptr(), bufs.wts.data_ptr(), bufs.h.data_ptr(),
                                              bufs.scratch.data_ptr(), bufs.counters.data_ptr(), num_sms, SILU, cl.stream_ptr()),
             "moe_decode_ffn_dense")
    torch.cuda.synchronize()
    return out, bufs.h.clone(), bufs.ids.clone(), bufs.wts.clone()


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    assert worst <= 1.0, f"{what}: error {err.max().item():.3g} is {worst:.3g} of its bound"


def check(x, out0, norm, gate, out, h, ids, wts, w13, w2, k, what, local=None):
    xd, nd = x.double(), norm.double()
    a = nd * xd / torch.sqrt((xd * xd).mean() + EPS)
    # routing: distinct ids; the float64 top-k wherever the k-th / (k+1)-th logits are clearly apart; weights softmax over them
    lg = gate.double() @ a
    top = torch.topk(lg, k + 1)
    assert len(set(ids.tolist())) == k
    if (top.values[k - 1] - top.values[k]).item() > 1e-4:
        assert set(ids.tolist()) == set(top.indices[:k].tolist()), f"{what}: routing differs from float64"
    sel = lg[ids.long()]
    wref = torch.softmax(sel, 0)
    assert (wts.double() - wref).abs().max().item() < 2.0 ** -16, f"{what}: routing weights"
    dx = torch.zeros_like(xd)
    tol = torch.zeros_like(xd)
    mag = torch.zeros_like(xd)
    for j, e in enumerate(ids.tolist()):
        if local is not None and not (local[0] <= e < local[0] + local[1]):
            assert (h[j] == 0).all(), f"{what}: slot {j} (expert {e}, not local) wrote h"
            continue
        W13 = w13[e].double()
        gu = W13 @ a
        egu = (C_DOT + REL_NORM) * (W13.abs() @ a.abs())
        g, u, eg, eu = gu[0::2], gu[1::2], egu[0::2], egu[1::2]
        sg = g * torch.sigmoid(g)
        h_ref = sg * u
        eh = 1.1 * eg * (u.abs() + eu) + sg.abs() * eu + REL_SILU * h_ref.abs() + 2.0 ** -23 * h_ref.abs()
        assert_within(h[j], h_ref, eh, f"{what}: h of slot {j} (expert {e})")
        W2 = w2[e].double()
        hd = h[j].double()
        y = W2 @ hd
        ey = C_DOT * (W2.abs() @ hd.abs())
        wt = wts[j].double()
        dx += wt * y
        tol += wt * ey
        mag += wt * y.abs()
    got = out.double() - out0.double()
    assert_within(got, dx, tol + (k + 2) * 2.0 ** -24 * (mag + out.double().abs()) + 1e-30, f"{what}: Δx")


@pytest.mark.parametrize("wtype", [1, 2], ids=["f32", "f16"])
@pytest.mark.parametrize("sms", ["device", 17])
@pytest.mark.parametrize("dim,ff,E,k", [SHAPE_TINY, SHAPE_30B, (2048, 384, 128, 8)])
def test_decode_ffn_dense(dim, ff, E, k, sms, wtype):
    """Three tokens through the same buffers (self-resetting counters); the expert sum is added to a non-zero `out`; each
    token twice, bitwise equal. sms = 17 gives 2 CTAs per routing slot at k = 8 instead of the engine's 16."""
    num_sms = _num_sms() if sms == "device" else sms
    w13, w2 = expert_weights(dim, ff, E, torch.float32 if wtype == 1 else torch.float16)
    bufs = Bufs(dim, ff, E, k, num_sms)
    for t in range(3):
        x, norm, gate = inputs(dim, E, 100 + t)
        out0 = x + 0.25 * torch.randn_like(x)
        what = f"{'f32' if wtype == 1 else 'f16'} {dim}/{ff}/{E}/{k} sms={num_sms} token {t}"
        out, h, ids, wts = ffn_call(wtype, x, out0, norm, gate, w13, w2, ff, k, num_sms, bufs)
        bufs.check(what)
        check(x, out0, norm, gate, out, h, ids, wts, w13, w2, k, what)
        out2, h2, ids2, wts2 = ffn_call(wtype, x, out0, norm, gate, w13, w2, ff, k, num_sms, bufs)
        bufs.check(what)
        assert torch.equal(out, out2) and torch.equal(h, h2) and torch.equal(ids, ids2) and torch.equal(wts, wts2), f"{what}: two runs differ"


@pytest.mark.parametrize("wtype", [1, 2], ids=["f32", "f16"])
def test_decode_ffn_dense_expert_parallel(wtype):
    """Two expert-parallel halves, each holding only its experts: slots routed to the other half write h = 0 and add nothing,
    each half is right on its own, and the halves sum to the full run within the f32 rounding of the two slot-order combines."""
    dim, ff, E, k = SHAPE_30B
    num_sms = _num_sms()
    w13, w2 = expert_weights(dim, ff, E, torch.float32 if wtype == 1 else torch.float16)
    bufs = Bufs(dim, ff, E, k, num_sms)
    x, norm, gate = inputs(dim, E, 7)
    zero = torch.zeros_like(x)
    full, _, ids, _ = ffn_call(wtype, x, zero, norm, gate, w13, w2, ff, k, num_sms, bufs)
    bufs.check("full")
    mag = bufs.scratch.double().abs().sum(0)   # sum over slots of |weight * product|: every partial sum of either side is below it
    half = E // 2
    assert any(e < half for e in ids.tolist()) and any(e >= half for e in ids.tolist()), "routing fell into one half"
    parts = []
    for first in (0, half):
        what = f"EP [{first}, {first + half})"
        out, h, ids_p, wts_p = ffn_call(wtype, x, zero, norm, gate, w13, w2, ff, k, num_sms, bufs, first, half)
        bufs.check(what)
        assert torch.equal(ids_p, ids)
        check(x, zero, norm, gate, out, h, ids_p, wts_p, w13, w2, k, what, local=(first, half))
        parts.append(out.double())
    # the products are bitwise the same in all three runs; each side sums them in slot order with at most k roundings of u * mag
    bound = 2 * (k + 2) * 2.0 ** -24 * mag + 1e-30
    assert_within(parts[0] + parts[1], full.double(), bound, "EP halves vs full")


# ---- engine and front ends on tiny Qwen3-MoE files -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def moe_dense_files(tmp_path_factory):
    from distributed_llama_b200.formats import quants
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model, write_synthetic_tokenizer
    root = tmp_path_factory.mktemp("moe_dense")
    cfg = get_config("tiny-qwen3-moe")
    tok = str(root / "tiny-qwen3-moe.t")
    write_synthetic_tokenizer(tok, cfg.vocab_size, style="chatml")
    out = {}
    for wt in ("f32", "f16", "q80"):
        path = str(root / f"tiny-qwen3-moe-{wt}.m")
        write_synthetic_model(path, cfg, weights_float_type=quants.parse_float_type(wt), seed=7)
        out[wt] = (path, tok)
    return out


@pytest.mark.parametrize("wt", ["f32", "f16", "q80"])
def test_engine_dense_moe_matches_oracle(moe_dense_files, wt):
    """Teacher-forced logits against the oracle without activation quantisation, at the dense files' tolerance (the bf16 KV
    cache); greedy device decoding follows the oracle's arg-max; a second engine reproduces the logits bit for bit."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    from distributed_llama_b200.runtime import Engine
    mf = ModelFile(moe_dense_files[wt][0])
    eng = Engine(load_device_weights(mf))
    assert eng.dense and not eng.mega and eng.max_batch == 1
    oracle = OracleModel(mf, act_quant="none", device="cuda")
    toks = [3, 17, 250, 9, 44, 101, 7, 300, 12, 5, 77]
    ref = oracle.forward(toks, 0)
    lg = eng.prefill(toks[:6], 0).clone()
    assert (lg - ref[5]).abs().max().item() < 2e-2
    rows = [lg]
    for i in range(6, len(toks)):
        lg = eng.step(toks[i], i).clone()
        rows.append(lg)
        assert (lg - ref[i]).abs().max().item() < 2e-2, i
    eng2 = Engine(load_device_weights(mf))
    again = [eng2.prefill(toks[:6], 0).clone()] + [eng2.step(toks[i], i).clone() for i in range(6, len(toks))]
    assert all(torch.equal(a, b) for a, b in zip(rows, again)), "two engines differ"
    out = eng.decode_greedy(toks[-1], len(toks) - 1, 6)
    tok, pos, want = toks[-1], len(toks) - 1, []
    for _ in range(3):
        tok = int(oracle.forward([tok], pos)[0].argmax())
        want.append(tok)
        pos += 1
    assert out[:3] == want


def test_dllama_inference_dense_moe(moe_dense_files):
    m, t = moe_dense_files["f16"]
    r = subprocess.run([os.path.join(ROOT, "dllama"), "inference", "--model", m, "--tokenizer", t, "--prompt", "Hello world, the model",
                        "--steps", "16", "--temperature", "0", "--seed", "1"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    assert "🔷️ Eval" in r.stdout and r.stdout.count("🔶 Pred") >= 4 and "RequiredMemory" in r.stdout


def test_dllama_api_dense_moe(moe_dense_files):
    import http.client
    import json
    import socket
    import time
    m, t = moe_dense_files["f16"]
    port = 21990 + os.getpid() % 1000
    p = subprocess.Popen([os.path.join(ROOT, "dllama-api"), "--model", m, "--tokenizer", t, "--port", str(port), "--host", "127.0.0.1",
                          "--temperature", "0"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        for _ in range(300):
            try:
                socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
                break
            except OSError:
                time.sleep(0.2)
        conn = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
        conn.request("POST", "/v1/chat/completions", json.dumps({"messages": [{"role": "user", "content": "Hello"}], "max_tokens": 8}),
                     {"Content-Type": "application/json"})
        resp = json.loads(conn.getresponse().read())
        assert resp["object"] == "chat.completion" and 1 <= resp["usage"]["completion_tokens"] <= 8
        assert resp["choices"][0]["message"]["role"] == "assistant"
    finally:
        p.terminate()
        p.communicate(timeout=30)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("mode", ["tp", "ep"])
def test_tp_check_dense_moe(mode):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29677", os.path.join(ROOT, "tools", "tp_check.py"), "tiny-qwen3-moe", mode, "f16"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert "TP_CHECK PASS" in r.stdout and f"moe_mode={mode}" in r.stdout, r.stdout[-3000:]
