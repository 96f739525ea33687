"""The persistent decode kernel's producer: its pacing (DL_MEGA_INFLIGHT, fills in flight per CTA) only changes when the weight bytes
arrive, never what is computed; with all-CTA tracing it records its stall counters per weight phase."""
import pytest
import torch

pytestmark = pytest.mark.gpu

PROMPT = [3, 17, 250, 9, 44, 101, 7]
INFLIGHT = [None, "2", "0"]         # the default (1), two fills, the whole ring


def _engine(tmp_models, name, monkeypatch, inflight):
    from distributed_llama_b200.formats import ModelFile
    from distributed_llama_b200.models.loader import load_device_weights
    from distributed_llama_b200.runtime import Engine
    if inflight is None:
        monkeypatch.delenv("DL_MEGA_INFLIGHT", raising=False)
    else:
        monkeypatch.setenv("DL_MEGA_INFLIGHT", inflight)
    eng = Engine(load_device_weights(ModelFile(tmp_models[name][0])))
    eng.enable_mega()                # the environment is read here
    eng.prefill(PROMPT[:-1], 0, want_logits=False)
    return eng


@pytest.mark.parametrize("name", ["tiny-llama31", "tiny-qwen3"])
def test_producer_pacing_does_not_change_results(tmp_models, monkeypatch, name):
    logits, eager, graph = {}, {}, {}
    for inflight in INFLIGHT:
        e = _engine(tmp_models, name, monkeypatch, inflight)
        logits[inflight] = e.step(PROMPT[-1], len(PROMPT) - 1).clone()
        assert e.mega_active
        e = _engine(tmp_models, name, monkeypatch, inflight)
        eager[inflight] = e.decode_greedy(PROMPT[-1], len(PROMPT) - 1, 40, use_graph=False)
        assert e.mega_active
        e = _engine(tmp_models, name, monkeypatch, inflight)
        graph[inflight] = e.decode_greedy(PROMPT[-1], len(PROMPT) - 1, 40, use_graph=True)
        assert e.mega_active
    base = INFLIGHT[0]
    for inflight in INFLIGHT[1:]:
        assert torch.equal(logits[inflight], logits[base]), f"logits differ with DL_MEGA_INFLIGHT={inflight}"
        assert eager[inflight] == eager[base], (inflight, eager[inflight], eager[base])
        assert graph[inflight] == graph[base], (inflight, graph[inflight], graph[base])
    assert eager[base] == graph[base]


def test_producer_stall_slots(tmp_models, monkeypatch):
    """All-CTA tracing: after the per-CTA consumer stamps, the producer records two stall counters per weight phase."""
    name = "tiny-qwen3"               # has phases in which some CTAs own no rows
    e = _engine(tmp_models, name, monkeypatch, None)
    e.enable_trace(1024, all_ctas=True)
    L = e.w.header.n_layers
    n_stamps = 18 * L + 5
    p0 = (n_stamps + 7) // 8 * 8
    n_prod = 2 * (4 * L + 1)
    rows = e.trace_buf.view(-1)[: e.num_sms * e.trace_stride].view(e.num_sms, e.trace_stride)
    assert e.trace_stride >= p0 + n_prod
    rows[:, n_stamps:] = -1           # sentinel: every producer slot must be overwritten, nothing past them
    e.step(PROMPT[-1], len(PROMPT) - 1)
    torch.cuda.synchronize()
    assert e.mega_active
    rows = rows.cpu()
    stamps = rows[:, :n_stamps]
    assert bool((stamps > 0).all()), "every CTA records all its consumer phase stamps"
    prod = rows[:, p0: p0 + n_prod]
    assert bool((prod >= 0).all()), "a producer slot was not written"
    assert bool((prod < stamps.max() - stamps.min() + 1).all()), "a stall counter exceeds the step"
    assert bool((rows[:, p0 + n_prod:] == -1).all()), "nothing is written past the producer slots"
