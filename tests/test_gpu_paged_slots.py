"""Paged KV-cache slots (--parallel-cache paged): the slots share every layer plane as one pool of 64-row pages.

* slotAttnKernel and the tensor-core slot prefill attention over paged slots against float64, bf16 and q80 caches, head dims 64
  and 128. Pages are mapped in reverse and in shuffled order, and every physical row a query must not see holds NaN (a NaN scale
  for q80), so a read through the wrong page, or past the chunk's last row, shows. Bounds: 2e-4 * max|V| for the decode tiles
  (tests/test_gpu_slots.py), (2^-9 + 2^-14) * max|V| + one bf16 ulp for the tensor-core prefill (tests/test_gpu_attn_prefill.py).
  Negative controls (a row read through its neighbour's table, every page off by one) must miss the bound by 10x or more.
* The engine: a slots step, slot prefill (K/V rows and the next step's logits) and slot_copy are bitwise the same in the split and
  the paged layout, and with contiguous and scattered pages: paging moves where rows live, not the arithmetic.
* A request longer than floor(context / slots) completes: its teacher-forced logits are within test_gpu_slots.py's oracle
  tolerance and its greedy tokens are those it draws with every other slot idle.
* The scheduler's pool rules on a small context: a blocked admission, eviction of idle caches (prefix reuse lost, then regained)
  and a completion cut for want of a page whose tokens are a prefix of the same request run alone.
"""
import math
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

N_SPLITS = 8
TOL_DECODE = 2e-4
TOL_TC = 2.0 ** -9 + 2.0 ** -14
PAGE = 64
# query lengths (rows seen): both sides of each page edge and of the split-count steps (a split per 64 rows, at most 8)
LENGTHS = [1, 63, 64, 65, 127, 128, 129, 192, 193, 448, 449, 512, 513]


def _bf16_ulp(x):
    a = x.abs().clamp_min(1e-30)
    return torch.pow(2.0, torch.floor(torch.log2(a)) - 7)


def _paged_pool(g, n_kv, hd, lengths, q8, order):
    """Planes [n_kv][rows][hd] full of NaN and one page table row per slot: slot b owns ceil(lengths[b] / 64) pages, in reverse
    physical order for slot 0 and shuffled for the others. Rows [0, lengths[b]) of a slot hold data; returns the planes, the table
    and each slot's logical K / V rows (float64, as the kernel reads them)."""
    pages = [-(-n // PAGE) for n in lengths]
    n_pages = sum(pages) + 1
    perm = torch.randperm(n_pages, generator=g).tolist()
    table = torch.zeros(len(lengths), max(pages), dtype=torch.int32)
    at = 0
    for b, n in enumerate(pages):
        mine = perm[at:at + n]
        at += n
        table[b, :n] = torch.tensor(sorted(mine, reverse=True) if (b == 0 or order == "reverse") else mine)
    rows = n_pages * PAGE
    if q8:
        kq = torch.randint(-127, 128, (n_kv, rows, hd), generator=g, dtype=torch.int8)
        vq = torch.randint(-127, 128, (n_kv, rows, hd), generator=g, dtype=torch.int8)
        ks = torch.full((n_kv, rows, hd // 32), float("nan"), dtype=torch.float16)
        vs = ks.clone()
    else:
        kq = torch.full((n_kv, rows, hd), float("nan"), dtype=torch.bfloat16)
        vq = kq.clone()
    logical = []
    for b, n in enumerate(lengths):
        phys = [int(table[b, r // PAGE]) * PAGE + r % PAGE for r in range(n)]
        if q8:
            ks[:, phys] = (torch.rand(n_kv, n, hd // 32, generator=g) * 0.01 + 0.002).half()
            vs[:, phys] = (torch.rand(n_kv, n, hd // 32, generator=g) * 0.02 + 0.002).half()
            kl = kq[:, phys].double() * ks[:, phys].double().repeat_interleave(32, -1)
            vl = vq[:, phys].double() * vs[:, phys].double().repeat_interleave(32, -1)
        else:
            kq[:, phys] = (torch.randn(n_kv, n, hd, generator=g) * 0.6).bfloat16()
            vq[:, phys] = torch.randn(n_kv, n, hd, generator=g).bfloat16()
            kl, vl = kq[:, phys].double(), vq[:, phys].double()
        logical.append((kl, vl))
    planes = (kq, vq, ks, vs) if q8 else (kq, vq, None, None)
    return planes, table, logical, rows


def _slot_attn(planes, table, rows, qkv, pos, n_heads, n_kv, hd, L):
    from distributed_llama_b200.ops import cuda_lib as cl
    B = len(pos)
    q_dim = n_heads * hd
    dev = [None if t is None else t.cuda().contiguous() for t in planes]
    ptr = [0 if t is None else t.data_ptr() for t in dev]
    td = table.cuda().contiguous()
    posd = torch.tensor(pos, dtype=torch.int32, device="cuda")
    qd = qkv.cuda().contiguous()
    partial = torch.zeros(B * n_heads * N_SPLITS * (hd + 2), device="cuda")
    counters = torch.zeros(B * n_kv, dtype=torch.int32, device="cuda")
    out = torch.full((B, q_dim), float("nan"), device="cuda")
    assert cl.lib().dl_slot_attn_paged(qd.data_ptr(), qkv.shape[1], posd.data_ptr(), ptr[0], ptr[1], ptr[2], ptr[3], td.data_ptr(),
                                       table.shape[1], rows, n_heads, n_kv, hd, L, N_SPLITS, B, 0, partial.data_ptr(),
                                       counters.data_ptr(), out.data_ptr(), q_dim, cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert int(counters.abs().sum()) == 0
    return out.cpu().double()


def _worst(got, logical, qkv, pos, n_heads, n_kv, hd, tol):
    """Largest err / bound over the rows and heads (inf for a non-finite output)."""
    kv_mul = n_heads // n_kv
    worst = 0.0
    for b, p in enumerate(pos):
        kl, vl = logical[b]
        n = p + 1
        for h in range(n_heads):
            q = qkv[b, h * hd:(h + 1) * hd].double()
            s = (kl[h // kv_mul, :n] @ q) / math.sqrt(hd)
            want = torch.softmax(s, 0) @ vl[h // kv_mul, :n]
            err = (got[b, h * hd:(h + 1) * hd] - want).abs().max().item()
            if not math.isfinite(err):
                return math.inf
            worst = max(worst, err / (tol * vl[h // kv_mul, :n].abs().max().item()))
    return worst


@pytest.mark.parametrize("q8", [False, True], ids=["bf16", "q80"])
@pytest.mark.parametrize("hd,kv_mul", [(64, 4), (128, 1), (128, 4)])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_paged_slot_attention_matches_float64(B, hd, kv_mul, q8):
    g = torch.Generator().manual_seed(B * 31 + hd + kv_mul + 7 * q8)
    n_kv = 2
    n_heads = n_kv * kv_mul
    qkv_dim = (n_heads + 2 * n_kv) * hd
    for first in range(0, len(LENGTHS), B):
        lengths = [LENGTHS[(first + b) % len(LENGTHS)] for b in range(B)]
        pos = [n - 1 for n in lengths]
        planes, table, logical, rows = _paged_pool(g, n_kv, hd, lengths, q8, "shuffled")
        qkv = torch.randn(B, qkv_dim, generator=g)
        L = table.shape[1] * PAGE
        got = _slot_attn(planes, table, rows, qkv, pos, n_heads, n_kv, hd, L)
        assert _worst(got, logical, qkv, pos, n_heads, n_kv, hd, TOL_DECODE) <= 1.0, lengths
        if B > 1:   # negative control: every row through its neighbour's table
            bad = _slot_attn(planes, table.roll(1, 0), rows, qkv, pos, n_heads, n_kv, hd, L)
            assert _worst(bad, logical, qkv, pos, n_heads, n_kv, hd, TOL_DECODE) >= 10.0
        # negative control: every page off by one
        bad = _slot_attn(planes, (table + 1) % (rows // PAGE), rows, qkv, pos, n_heads, n_kv, hd, L)
        assert _worst(bad, logical, qkv, pos, n_heads, n_kv, hd, TOL_DECODE) >= 10.0


def _prefill(planes, table, rows, qkv, T, p0, n_heads, n_kv, hd):
    from distributed_llama_b200.ops import cuda_lib as cl
    dev = [None if t is None else t.cuda().contiguous() for t in planes]
    ptr = [0 if t is None else t.data_ptr() for t in dev]
    td = table.cuda().contiguous()
    qd = qkv.cuda().contiguous()
    out = torch.full((T, n_heads * hd), float("nan"), dtype=torch.bfloat16, device="cuda")
    assert cl.lib().dl_attn_prefill_tc_paged(qd.data_ptr(), qkv.shape[1], T, p0, n_heads, n_kv, hd, rows, ptr[0], ptr[1], ptr[2], ptr[3],
                                             td.data_ptr(), out.data_ptr(), n_heads * hd, cl.stream_ptr()) == 0
    torch.cuda.synchronize()
    return out.cpu().double()


def _prefill_worst(got, kl, vl, qkv, T, p0, n_heads, n_kv, hd):
    kv_mul = n_heads // n_kv
    worst = 0.0
    for t in range(T):
        n = p0 + t + 1
        for h in range(n_heads):
            q = qkv[t, h * hd:(h + 1) * hd].double()
            want = torch.softmax((kl[h // kv_mul, :n] @ q) / math.sqrt(hd), 0) @ vl[h // kv_mul, :n]
            row = got[t, h * hd:(h + 1) * hd]
            if not torch.isfinite(row).all():
                return math.inf
            bound = TOL_TC * vl[h // kv_mul, :n].abs().max().item() + _bf16_ulp(want)
            worst = max(worst, ((row - want).abs() / bound).max().item())
    return worst


@pytest.mark.parametrize("q8", [False, True], ids=["bf16", "q80"])
@pytest.mark.parametrize("hd,kv_mul", [(64, 4), (128, 1), (128, 4)])
@pytest.mark.parametrize("T,p0", [(1, 0), (7, 63), (64, 64), (65, 0), (191, 65), (192, 1), (256, 0), (129, 127)])
def test_paged_prefill_attention_matches_float64(T, p0, hd, kv_mul, q8):
    g = torch.Generator().manual_seed(T * 13 + p0 + hd + kv_mul + 5 * q8)
    n_kv = 2
    n_heads = n_kv * kv_mul
    qkv = torch.randn(T, (n_heads + 2 * n_kv) * hd, generator=g)
    # the slot's rows [0, p0 + T) hold data; its last page past p0 + T and every other page hold NaN
    planes, table, logical, rows = _paged_pool(g, n_kv, hd, [p0 + T], q8, "reverse")
    kl, vl = logical[0]
    if q8:   # the q80 producer widens q * d to bf16 for the tensor cores (exact in f32: 8-bit times 11-bit significands)
        kl, vl = kl.float().bfloat16().double(), vl.float().bfloat16().double()
    got = _prefill(planes, table, rows, qkv, T, p0, n_heads, n_kv, hd)
    assert _prefill_worst(got, kl, vl, qkv, T, p0, n_heads, n_kv, hd) <= 1.0
    bad = _prefill(planes, (table + 1) % (rows // PAGE), rows, qkv, T, p0, n_heads, n_kv, hd)
    assert _prefill_worst(bad, kl, vl, qkv, T, p0, n_heads, n_kv, hd) >= 10.0


# ---- the engine -----------------------------------------------------------------------------------------------------------------

def _engine(tmp_models, name, slots, layout, kv="bf16", max_prefill=192):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    eng = Engine(load_device_weights(ModelFile(tmp_models[name][0])), kv_cache_float_type=kv, max_prefill=max_prefill)
    eng.set_slots(slots, layout)
    return eng


def _slot_rows(eng, slot, n):
    """Rows [0, n) of slot `slot` of every layer's K and V caches (and q80 scales), in logical order."""
    h_kv, hd = eng.k_cache[0].shape[0], eng.k_cache[0].shape[-1]
    out = []
    for l in range(len(eng.k_cache)):
        for cache, sc in ((eng.k_cache[l], eng.k_scale[l]), (eng.v_cache[l], eng.v_scale[l])):
            if eng.paged:
                pages = eng.slot_pages(slot)
                idx = torch.tensor([pages[r // PAGE] * PAGE + r % PAGE for r in range(n)], device=cache.device)
                planes = [cache.view(h_kv, -1, hd)]
                if sc is not None:
                    planes.append(sc[:h_kv * eng.seq_len * hd // 32].view(h_kv, -1, hd // 32))
                out += [p[:, idx].clone() for p in planes]
            else:
                L = eng.slot_len
                planes = [cache.view(-1)[slot * h_kv * L * hd:(slot + 1) * h_kv * L * hd].view(h_kv, L, hd)]
                if sc is not None:
                    planes.append(sc[slot * h_kv * L * hd // 32:(slot + 1) * h_kv * L * hd // 32].view(h_kv, L, hd // 32))
                out += [p[:, :n].clone() for p in planes]
    return out


def _scatter(eng, slots, rows):
    """Paged: reserves `rows` rows for each slot one page at a time, round robin, so that the slots' pages interleave."""
    for r in range(PAGE, rows + PAGE, PAGE):
        for s in slots:
            assert eng.slot_reserve(s, min(r, rows))


@pytest.mark.parametrize("kv", ["bf16", "q80"])
@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_step_split_paged_and_scattered_are_bitwise_equal(tmp_models, name, kv):
    N, steps = 4, 12
    engines = {m: _engine(tmp_models, name, N, "split" if m == "split" else "paged", kv) for m in ("split", "paged", "scattered")}
    L = engines["split"].slot_len
    prompts = [[(11 * b + 7 * i + 3) % 500 + 1 for i in range(5 + 9 * b)] for b in range(N)]
    for m, eng in engines.items():
        if m == "paged":
            for b in range(N):
                assert eng.slot_reserve(b, L)
        elif m == "scattered":
            _scatter(eng, range(N), L)
        for b in range(N):
            eng.slot_prefill(b, prompts[b][:-1], 0)
    assert engines["paged"].slot_pages(1) == list(range(L // PAGE, 2 * L // PAGE))
    if L > PAGE:
        assert engines["scattered"].slot_pages(1)[:2] == [1, N + 1]
    logits = {m: [] for m in engines}
    for m, eng in engines.items():
        tokens = [p[-1] for p in prompts]
        pos = [len(p) - 1 for p in prompts]
        for j in range(steps):
            active = [not (b == 2 and j % 3 == 0) for b in range(N)]
            logits[m].append(eng.slots_forward(tokens, pos, active).clone())
            for b in range(N):
                if active[b]:
                    tokens[b] = int(logits[m][-1][b].argmax())
                    pos[b] += 1
    for j in range(steps):
        assert torch.equal(logits["split"][j], logits["paged"][j]), j
        assert torch.equal(logits["paged"][j], logits["scattered"][j]), j
    for b in range(N):
        n = len(prompts[b]) + steps - 1
        for x, y, z in zip(_slot_rows(engines["split"], b, n), _slot_rows(engines["paged"], b, n), _slot_rows(engines["scattered"], b, n)):
            assert torch.equal(x, y) and torch.equal(y, z)


@pytest.mark.parametrize("kv", ["bf16", "q80"])
@pytest.mark.parametrize("T", [1, 7, 64, 191, 192, 256])
def test_slot_prefill_and_copy_split_equals_paged(tmp_models, T, kv):
    """Prompt chunks of T tokens after a first chunk that leaves p0 off a page edge; K/V rows and the next step's logits bitwise
    equal in both layouts; slot_copy of the prompt rows likewise. (256 tokens fill a split slot of the 512-row context: rows only.)"""
    name, N = "tiny-llama31", 2
    p0 = 0 if T == 256 else 5 + T % 3
    step = T < 256
    prompt = [(13 * i + 5) % 500 + 1 for i in range(p0 + T + 1)]
    res = {}
    for layout in ("split", "paged"):
        eng = _engine(tmp_models, name, N, layout, kv, max_prefill=256)
        if layout == "paged":
            _scatter(eng, [1, 0], p0 + T + step)
        if p0:
            eng.slot_prefill(0, prompt[:p0], 0)
        eng.slot_prefill(0, prompt[p0:p0 + T], p0)
        eng.slot_copy(0, 1, p0 + T)
        lg = eng.slots_forward([prompt[-1]] * N, [p0 + T] * N, [True] * N).clone() if step else None
        res[layout] = (lg, _slot_rows(eng, 0, p0 + T + step), _slot_rows(eng, 1, p0 + T + step))
    if step:
        assert torch.equal(res["split"][0], res["paged"][0])
        assert torch.equal(res["paged"][0][0], res["paged"][0][1])   # the copy holds the same rows
    for i in (1, 2):
        for x, y in zip(res["split"][i], res["paged"][i]):
            assert torch.equal(x, y)


def test_request_beyond_split_length_completes(tmp_models):
    """Paged, 4 slots of a 512-row context: one request runs 100 prompt tokens + 250 generated ones (past floor(512 / 4) = 128)
    while the other slots run short requests. Its greedy tokens equal those it draws alone; its teacher-forced logits are within
    test_gpu_slots.py's oracle tolerance."""
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.models.reference import OracleModel
    from distributed_llama_b200.runtime import Engine
    name, N, P, gen = "tiny-llama31", 4, 99, 250
    prompt = [(17 * i + 3) % 500 + 1 for i in range(P + 1)]

    def run(busy):
        eng = _engine(tmp_models, name, N, "paged")
        assert eng.slot_len == 512
        assert eng.slot_reserve(0, P + 1)
        eng.slot_prefill(0, prompt[:-1], 0)
        others = [[(5 * b + 11 * i) % 500 + 1 for i in range(20)] for b in range(N)]
        if busy:
            for b in range(1, N):
                assert eng.slot_reserve(b, 64)
                eng.slot_prefill(b, others[b][:-1], 0)
        tokens = [prompt[-1]] + [others[b][-1] for b in range(1, N)]
        pos = [P] + [19] * (N - 1)
        out, lgs = [], []
        for j in range(gen):
            active = [True] + [busy and pos[b] < 63 for b in range(1, N)]
            for b in range(1, N):
                if not active[b]:
                    eng.slot_release(b)                     # a finished request's pages go back to the pool
            assert eng.slot_reserve(0, pos[0] + 1)
            lg = eng.slots_forward(tokens, pos, active).clone()
            lgs.append(lg[0])
            nxt = lg.argmax(-1).tolist()
            out.append(nxt[0])
            for b in range(N):
                if active[b]:
                    tokens[b], pos[b] = nxt[b], pos[b] + 1
        return out, lgs

    alone, _ = run(False)
    together, lgs = run(True)
    assert together == alone
    # teacher-forced against OracleModel at test_gpu_slots.py's tolerance: within max(0.06, the single-sequence engine's own
    # distance + 0.03)
    mf = ModelFile(tmp_models[name][0])
    seq = prompt + together
    ref = OracleModel(mf, act_quant="q80", device="cuda").forward(seq[:P + gen], 0)[P:]
    one = Engine(load_device_weights(mf))
    one.tc_min_tokens = 1
    one.prefill(prompt[:-1], 0, want_logits=False)
    for j in range(gen):
        single = one.step(seq[P + j], P + j)
        err = (lgs[j] - ref[j]).abs().max().item()
        base = (single - ref[j]).abs().max().item()
        assert err < max(0.06, base + 0.03), (j, err, base)


# ---- the scheduler's pool rules on the GPU ----------------------------------------------------------------------------------------

class _Req:
    """A SlotRequest over a token prompt: greedy, no end of sequence, the slot's cache a token prefix."""

    def __init__(self, sched_log, name, prompt, max_tokens, caches):
        from distributed_llama_b200.api import SlotRequest
        self.__class__ = type("R", (_Req, SlotRequest), {})
        self.log, self.name, self.prompt, self.max_tokens, self.caches = sched_log, name, prompt, max_tokens, caches
        self.temperature, self.n, self.seed = 0.0, 1, 1
        self.out, self.done = None, threading.Event()

    def cached_prefix(self, slot):
        c = self.caches[slot]
        return len(c) if c and len(c) < len(self.prompt) and self.prompt[:len(c)] == c else 0

    def prompt_len(self, slot):
        return len(self.prompt) - 1

    def prepare(self, slot):
        start = self.cached_prefix(slot)
        self.log.append(("admit", self.name, slot, start))
        self.caches[slot] = list(self.prompt)
        return self.prompt[start:-1], start, self.prompt[-1], len(self.prompt) - 1

    def on_token(self, i, tok):
        return False

    def finish(self, out, slots, P):
        self.caches[slots[0]] = self.prompt + out[0][:-1]
        self.out = out[0]
        self.log.append(("finish", self.name))
        self.done.set()

    def fail(self, e, slots):
        self.log.append(("fail", self.name, str(e)))
        self.done.set()


class _Served:
    """A SlotScheduler over `sess` on its own thread; on_evict forgets the slot's cache and records the slot."""

    def __init__(self, sess, caches):
        from distributed_llama_b200.api import SlotScheduler
        self.evicted = []

        def on_evict(s):
            self.evicted.append(s)
            caches[s] = None

        self.sched = SlotScheduler(sess, lambda: 1, on_evict=on_evict)
        self.thread = threading.Thread(target=self.sched.run, daemon=True)
        self.thread.start()

    def run(self, *reqs):
        for r in reqs:
            self.sched.submit(r)
        for r in reqs:
            assert r.done.wait(120), r.name

    def stop(self):
        self.sched.stop()
        self.thread.join(30)


def test_pool_rules(tmp_models):
    """Context 256 = 4 pages, 2 slots. y and x take 2 pages each; then a 130-token prompt needs all 4 and evicts x's idle cache
    (y's slot is the one it takes); x's follow-up has lost its prefix and waits for a's pages (blocked admission); the follow-up of
    that one regains its prefix. Two long completions that together outgrow the pool: one is cut, and its tokens are a prefix of
    the same request run alone."""
    from distributed_llama_b200.api import InferenceSession
    path = tmp_models["tiny-llama31"][0]
    sess = InferenceSession(path, max_seq_len=256, parallel=2, parallel_cache="paged")
    assert sess.slot_len == 256 and sess.free_pages() == 4
    log, caches = [], [None, None]
    srv = _Served(sess, caches)
    y = _Req(log, "y", [(7 * i + 1) % 500 + 1 for i in range(20)], 60, caches)
    x = _Req(log, "x", [(5 * i + 2) % 500 + 1 for i in range(20)], 60, caches)
    srv.run(y, x)
    assert [e[2] for e in log if e[0] == "admit"] == [0, 1]
    a = _Req(log, "a", [(3 * i + 5) % 500 + 1 for i in range(130)], 20, caches)
    x2 = _Req(log, "x2", x.prompt + x.out + [9, 9], 4, caches)
    srv.run(a, x2)
    assert srv.evicted == [1], log
    assert [e for e in log if e[:2] == ("admit", "x2")][0][3] == 0          # x's cache was evicted: no prefix reuse
    assert log.index(("finish", "a")) < [i for i, e in enumerate(log) if e[:2] == ("admit", "x2")][0]   # x2 waited for a's pages
    x3 = _Req(log, "x3", x2.prompt + x2.out + [7], 4, caches)
    srv.run(x3)
    assert [e for e in log if e[:2] == ("admit", "x3")][0][3] == len(x2.prompt + x2.out[:-1])   # x2's cache is reused
    srv.stop()
    # the cut: two 20-token prompts, each asking for 230 tokens; 4 pages cannot hold both
    log2, caches2 = [], [None, None]
    srv = _Served(InferenceSession(path, max_seq_len=256, parallel=2, parallel_cache="paged"), caches2)
    c = _Req(log2, "c", [(3 * i + 4) % 500 + 1 for i in range(20)], 230, caches2)
    d = _Req(log2, "d", [(11 * i + 6) % 500 + 1 for i in range(20)], 230, caches2)
    srv.run(c, d)
    srv.stop()
    lens = sorted([len(c.out), len(d.out)])
    assert lens[0] < 230 and lens[1] == 230, lens
    cut = c if len(c.out) < 230 else d
    srv = _Served(InferenceSession(path, max_seq_len=256, parallel=2, parallel_cache="paged"), [None, None])
    solo = _Req([], "solo", cut.prompt, 230, [None, None])
    srv.run(solo)
    srv.stop()
    assert solo.out[:len(cut.out)] == cut.out


@pytest.mark.parametrize("kv", ["bf16", "q80"])
def test_slot_copy_reserves_the_destination(tmp_models, kv):
    """slot_copy into a slot that holds no pages reserves them itself (lowest free first) and copies the rows bitwise; when the pool
    is short it fails with -68 and changes nothing."""
    eng = _engine(tmp_models, "tiny-llama31", 2, "paged", kv)   # 512 rows: 8 pages
    prompt = [(13 * i + 5) % 500 + 1 for i in range(150)]
    assert eng.slot_reserve(0, 150)
    eng.slot_prefill(0, prompt, 0)
    eng.slot_copy(0, 1, 150)
    assert eng.slot_pages(1) == [3, 4, 5] and eng.free_pages() == 2
    for x, y in zip(_slot_rows(eng, 0, 150), _slot_rows(eng, 1, 150)):
        assert torch.equal(x, y)
    eng.slot_release(1)
    assert eng.slot_reserve(0, 7 * PAGE) and eng.free_pages() == 1
    with pytest.raises(RuntimeError, match="-68"):
        eng.slot_copy(0, 1, 150)
    assert eng.slot_pages(1) == [] and eng.free_pages() == 1
