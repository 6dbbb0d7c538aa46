"""GPU, f4: deep profile -- per-layer forward / backward device timers and activation sizes
(K1 / K2 with a layer id) next to CUDA events around the same layers, and next to the
reference's own layer hooks when oracle/_ref is present."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture()
def deep(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    monkeypatch.setenv("TRACEML_PROFILE", "deep")
    from traceml_b200.instrumentation import layers

    layers.reset()
    yield layers
    layers.reset()


def _model():
    return torch.nn.Sequential(torch.nn.Linear(1024, 4096), torch.nn.GELU(), torch.nn.Linear(4096, 1024),
                               torch.nn.LayerNorm(1024), torch.nn.Linear(1024, 16)).cuda()


def test_layer_records_through_the_public_api(deep):
    import traceml_b200 as traceml
    from traceml_b200 import runtime
    from traceml_b200.runtime import reset_trace_session_state

    reset_trace_session_state(0)
    traceml.init(mode="auto")
    model = _model()
    traceml.trace_model_instance(model)              # gate: TRACEML_PROFILE=deep
    prof = deep.profile_of(model)
    assert prof is not None and prof.names == ["0", "1", "2", "3", "4"]
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    n_steps, batch = 6, 256
    for _ in range(n_steps):
        x = torch.randn(batch, 1024, device="cuda")
        with traceml.trace_step(model):
            out = model(x)
            out = out + model[4](model[3](torch.randn(batch, 1024, device="cuda")))   # layers 3, 4 called twice
            out.sum().backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    recs = prof.drain()
    assert recs.shape == (n_steps, 5)
    first = runtime.get_trace_session_state().step - n_steps + 1
    assert [int(r["step"][0]) for r in recs] == list(range(first, first + n_steps))
    assert (recs["fwd_calls"][:, :3] == 1).all() and (recs["fwd_calls"][:, 3:] == 2).all()
    assert (recs["bwd_calls"][:, 1:3] == 1).all() and (recs["bwd_calls"][:, 3:] == 2).all()
    assert (recs["fwd_ns"] > 0).all() and (recs["bwd_ns"][:, 1:] > 0).all()
    # activation bytes are exact: fp32 outputs of known shapes, summed over the calls of the step
    assert (recs["fwd_bytes"][:, 0] == batch * 4096 * 4).all() and (recs["fwd_bytes"][:, 4] == 2 * batch * 16 * 4).all()
    # the big matmuls dominate the cheap activation / norm layers
    assert np.median(recs["fwd_ns"][:, 0]) > np.median(recs["fwd_ns"][:, 1])
    rows = prof.wire_rows(recs)
    r0 = rows["layer_forward_time"][0]
    assert set(r0) == {"seq", "ts", "model_id", "step", "device", "layers", "cpu_ms", "gpu_ms", "n_calls"}
    assert r0["layers"] == prof.names and r0["n_calls"] == [1, 1, 1, 2, 2] and r0["device"] == "cuda:0"
    assert len(rows["layer_backward_time"]) == n_steps and len(rows["layer_forward_memory"]) == n_steps


def test_layer_timers_bracketed_by_cuda_events(deep):
    """Same physical statement as for the phase stamps: an event pair recorded INSIDE the layer
    region cannot exceed the layer's device duration (2 us + 1 %)."""
    from traceml_b200.engine import Engine

    eng = Engine(device=0, ring_slots=64)
    big = torch.nn.Linear(4096, 4096).cuda()
    model = torch.nn.Sequential(big).cuda()
    prof = deep.LayerProfile(eng, model, backward=False)
    evs = []

    def pre(m, a):
        e = torch.cuda.Event(enable_timing=True); e.record(); evs.append([e])

    def post(m, a, o):
        e = torch.cuda.Event(enable_timing=True); e.record(); evs[-1].append(e)

    big.register_forward_pre_hook(pre)     # registered AFTER the profile's hooks: inside the layer region
    big.register_forward_hook(post, prepend=True)
    x = torch.randn(2048, 4096, device="cuda")
    for step in range(1, 41):
        for _ in range(1 + step % 3):
            model(x)
        prof.commit(step)
    torch.cuda.synchronize()
    recs = prof.drain()
    assert recs.shape == (40, 1)
    k = 0
    for step in range(1, 41):
        calls = 1 + step % 3
        inner_us = sum(a.elapsed_time(b) * 1000.0 for a, b in evs[k:k + calls])
        k += calls
        mine_us = float(recs["fwd_ns"][step - 1, 0]) / 1000.0
        assert int(recs["fwd_calls"][step - 1, 0]) == calls
        assert mine_us >= inner_us - (2.0 * calls + 0.01 * mine_us), (step, mine_us, inner_us)
        assert mine_us <= inner_us + 30.0 * calls + 0.02 * mine_us, (step, mine_us, inner_us)
    prof.detach()
    eng.close()


def test_layer_times_next_to_the_reference_hooks(deep):
    """The UNMODIFIED reference's layer forward timing hooks (CUDA events resolved by its sampler
    helper) on the same model in the same steps."""
    if not os.path.isdir(os.path.join(REF, "traceml")):
        pytest.skip("oracle/_ref is not present")
    os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from traceml.instrumentation.hooks.layer_forward_time_hooks import (attach_layer_forward_time_hooks,
                                                                        flush_layer_forward_time_buffers,
                                                                        get_layer_forward_time_queue)

    from traceml_b200.engine import Engine

    eng = Engine(device=0, ring_slots=64)
    model = _model()
    attach_layer_forward_time_hooks(model)                                  # the reference's: inner pair
    prof = deep.LayerProfile(eng, model, backward=False, outermost=True)     # ours brackets them
    x = torch.randn(512, 1024, device="cuda")
    n = 30
    for step in range(1, n + 1):
        model(x)
        prof.commit(step)
        flush_layer_forward_time_buffers(model, step)
    torch.cuda.synchronize()
    recs = prof.drain()
    q = get_layer_forward_time_queue()
    ref_steps = []
    while not q.empty():
        ref_steps.append(q.get_nowait())
    assert len(ref_steps) == n == recs.shape[0]
    gaps = []
    for row, ev in zip(recs, ref_steps):
        assert int(row["step"][0]) == ev.step
        by_name = {}
        for le in ev.layers:
            assert le.try_resolve()
            by_name[le.layer_name] = by_name.get(le.layer_name, 0.0) + le.gpu_duration_ms * 1000.0
        for i, name in enumerate(prof.names):
            mine = float(row["fwd_ns"][i]) / 1000.0
            assert mine >= by_name[name] - (2.0 + 0.01 * mine), (name, mine, by_name[name])
            gaps.append(mine - by_name[name])
    # ours is the OUTER pair: the reference's own hook work (two event records, Python) sits between
    # our stamps and shows up as device idle time on this tiny model (a descheduled host thread makes
    # single outliers: the bound is on the median)
    assert np.median(gaps) < 150.0, np.percentile(gaps, [0, 50, 90, 100])
    prof.detach()
    eng.close()
