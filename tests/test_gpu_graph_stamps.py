"""GPU: regions captured into a CUDA graph (``trace_graph``, tml_graph_*) are stamped on every
replay, land in the step that runs the replay, and the graph keeps the device state it writes to
alive.  The checks are physical (CUDA events recorded inside the same graph) and exact on counts
and step attribution."""
import gc
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FWD, BWD, OPT = 2, 3, 4


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _lib():
    from traceml_b200 import _abi

    return _abi.lib()


def _spin_matmul(a, k):
    for _ in range(k):
        a = a @ a
        a = a / a.norm()
    return a


def _timed_event():
    return torch.cuda.Event(enable_timing=True, external=True)


def _wait_graph_refs(value, timeout_s=10.0):
    """CUDA runs a user object's destructor after the graph's work is done, from its own thread."""
    lib = _lib()
    t0 = time.monotonic()
    while lib.tml_graph_refs() != value and time.monotonic() - t0 < timeout_s:
        gc.collect()
        time.sleep(0.01)
    return int(lib.tml_graph_refs())


def _capture_stamped(eng, phase, body, events=None):
    """A graph holding one region of `phase` around `body()`; `events` = (outer0, outer1, inner0,
    inner1) recorded just outside and just inside the region."""
    lib = _lib()
    g = torch.cuda.CUDAGraph()
    out = {}
    with torch.cuda.graph(g):  # capture_error_mode="global": the capture-time calls must not invalidate it
        s = torch.cuda.current_stream().cuda_stream
        if events:
            events[0].record()
        slot = lib.tml_graph_phase_begin(eng._h, phase, s)
        assert slot == 0, slot
        if events:
            events[2].record()
        out["y"] = body()
        if events:
            events[3].record()
        assert lib.tml_graph_phase_end(eng._h, phase, slot, s) == 0
        if events:
            events[1].record()
    return g, out


# ------------------------------------------------------------------------------------------- 1
def test_graph_stamp_bracketed_by_events_in_the_graph(cuda):
    """Per replay: inner <= stamp <= outer within 2 us + 1 % (SURVEY 8d); means within 0.5 %."""
    from traceml_b200.engine import Engine

    eng = Engine(device=0, ring_slots=1024)
    mats = [torch.randn(n, n, device="cuda") for n in (256, 512, 1024, 2048)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up: cuBLAS picks its kernels before the capture
        for m in mats:
            _spin_matmul(m, 3)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graphs = []
    for i, m in enumerate(mats):
        evs = tuple(_timed_event() for _ in range(4))
        g, _ = _capture_stamped(eng, FWD, lambda m=m, k=1 + i: _spin_matmul(m, k), evs)
        graphs.append((g, evs))
    s = torch.cuda.current_stream().cuda_stream
    n = 200
    outer, inner = np.zeros(n), np.zeros(n)
    for step in range(1, n + 1):
        g, evs = graphs[step % len(graphs)]
        g.replay()
        assert eng.step_commit(step, 0, 0, 0, 0.0, s) == 0
        torch.cuda.synchronize()  # the graph's events are re-recorded by the next replay
        outer[step - 1] = evs[0].elapsed_time(evs[1]) * 1000.0
        inner[step - 1] = evs[2].elapsed_time(evs[3]) * 1000.0
    recs, dropped = eng.drain()
    assert dropped == 0 and len(recs) == n
    assert list(recs["step"]) == list(range(1, n + 1))
    assert (recs["n_calls"][:, FWD] == 1).all() and (recs["gpu_mask"] == 1 << FWD).all()
    stamp = recs["dur_ns"][:, FWD].astype(np.float64) / 1000.0
    tol = 2.0 + 0.01 * stamp
    hist = {"outer_minus_stamp": np.percentile(outer - stamp, [0, 50, 100]).tolist(),
            "stamp_minus_inner": np.percentile(stamp - inner, [0, 50, 100]).tolist(),
            "stamp_us": np.percentile(stamp, [0, 50, 100]).tolist()}
    assert (stamp <= outer + tol).all(), hist
    assert (stamp >= inner - tol).all(), hist
    assert inner.mean() * 0.995 - 2.0 <= stamp.mean() <= outer.mean() * 1.005 + 2.0, hist
    del graphs
    eng.close()


# ------------------------------------------------------------------------------------------- 2
def test_replays_land_in_the_step_that_runs_them(cuda):
    """Step k replays the graph r_k in {0..3} times with the host > 8 commits ahead of the GPU:
    n_calls == r_k exactly, the phase's gpu_mask bit is set exactly when r_k > 0, the duration
    lies inside the bracket of the step's replays, and a host-launched region of the same phase
    in the same step adds its call and its duration."""
    from traceml_b200.engine import Engine

    eng = Engine(device=0, ring_slots=256)
    m = torch.randn(1024, 1024, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _spin_matmul(m, 3)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    evs = tuple(_timed_event() for _ in range(4))
    g, _ = _capture_stamped(eng, FWD, lambda: _spin_matmul(m, 4), evs)
    s = torch.cuda.current_stream()
    inner_us = []
    for _ in range(8):  # the region's own device time, replay by replay
        g.replay()
        torch.cuda.synchronize()
        inner_us.append(evs[2].elapsed_time(evs[3]) * 1000.0)
    eng.reset()
    rng = np.random.default_rng(7)
    n = 40
    reps = rng.integers(0, 4, n)
    host_region = [bool(r > 0 and k % 3 == 0) for k, r in enumerate(reps)]
    brackets = []
    torch.cuda._sleep(int(0.1 * 1.9e9))  # ~0.1 s of device time ahead of the loop
    for k in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(int(reps[k])):
            g.replay()
        if host_region[k]:
            slot = eng.phase_begin(FWD, s.cuda_stream)
            assert slot >= 0
            _spin_matmul(m, 2)
            assert eng.phase_end(FWD, slot, s.cuda_stream) == 0
        e1.record()
        brackets.append((e0, e1))
        assert eng.step_commit(k + 1, 0, 0, 0, 0.0, s.cuda_stream) == 0
    assert not s.query(), "the queued work finished before the loop did: the host was not ahead"
    torch.cuda.synchronize()
    recs, dropped = eng.drain()
    assert dropped == 0 and len(recs) == n
    assert list(recs["step"]) == list(range(1, n + 1))
    want_calls = reps + np.array(host_region, dtype=np.int64)
    assert list(recs["n_calls"][:, FWD]) == list(want_calls)
    assert list((recs["gpu_mask"] >> FWD) & 1) == [int(r > 0) for r in reps]
    dur = recs["dur_ns"][:, FWD].astype(np.float64) / 1000.0
    outer = np.array([e0.elapsed_time(e1) * 1000.0 for e0, e1 in brackets])
    lo = reps * min(inner_us) * 0.9
    assert (dur <= outer + 2.0 + 0.01 * outer).all(), (dur.tolist(), outer.tolist())
    assert (dur >= lo).all(), (dur.tolist(), lo.tolist())
    assert (dur[reps == 0] == 0).all()
    del g
    eng.close()


# ------------------------------------------------------------------------------------------- 3
def _graph_model():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(256, 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 10)).cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)
    x = torch.randn(128, 256, device="cuda")
    y = torch.randint(0, 10, (128,), device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up on a side stream, as torch's whole-network capture recipe
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(x), y).backward()
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    opt.zero_grad(set_to_none=True)
    return model, opt, x, y


def _capture_step(model, opt, x, y):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        torch.nn.functional.cross_entropy(model(x), y).backward()
        opt.step()
    return g


def test_whole_step_graph_through_the_public_api(cuda):
    import traceml_b200 as traceml
    from helpers import build_vs_row_oracles
    from traceml_b200 import runtime
    from traceml_b200.runtime import reset_trace_session_state

    traceml.init(mode="auto")
    eng = runtime.get_engine()
    model, opt, x, y = _graph_model()
    with traceml.trace_graph(model):
        g = _capture_step(model, opt, x, y)
    torch.cuda.synchronize()
    eng.reset()          # the warm-up's optimizer regions went into the open step: start clean
    reset_trace_session_state(0)
    n = 64
    evs = []
    for i in range(n):
        with traceml.trace_step(model):
            x.copy_(torch.randn(128, 256, device="cuda"))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            evs.append((e0, e1))
    torch.cuda.synchronize()
    recs, dropped = eng.drain()
    assert dropped == 0 and list(recs["step"]) == list(range(1, n + 1))
    for p in (FWD, BWD, OPT):
        assert (recs["n_calls"][:, p] == 1).all(), (p, recs["n_calls"][:, p])
        assert (recs["dur_ns"][:, p] > 0).all(), p
    assert ((recs["gpu_mask"] >> FWD) & 0b111 == 0b111).all()
    compute = recs["dur_ns"][:, [FWD, BWD, OPT]].sum(axis=1).astype(np.float64) / 1000.0
    replay_us = np.array([a.elapsed_time(b) * 1000.0 for a, b in evs])
    assert (compute <= replay_us + 2.0 + 0.01 * replay_us).all(), (compute.tolist(), replay_us.tolist())
    build_vs_row_oracles(eng, recs, n)   # the Step Time / Step Memory sections final_summary() builds

    # today's behaviour, kept: a graph captured outside trace_graph records no compute regions
    model2, opt2, x2, y2 = _graph_model()
    g2 = _capture_step(model2, opt2, x2, y2)
    torch.cuda.synchronize()
    eng.reset()          # the warm-up's optimizer regions and the capture's host-clock one
    for _ in range(8):
        with traceml.trace_step(model2):
            g2.replay()
    torch.cuda.synchronize()
    recs2, _ = eng.drain()
    assert len(recs2) == 8
    assert (recs2["n_calls"][:, [FWD, BWD, OPT]] == 0).all(), recs2["n_calls"]
    del g, g2


# ------------------------------------------------------------------------------------------- 4
@pytest.fixture()
def deep(monkeypatch, cuda):
    monkeypatch.setenv("TRACEML_PROFILE", "deep")
    from traceml_b200.instrumentation import layers

    layers.reset()
    yield layers
    layers.reset()


def test_deep_profile_in_a_graph(deep):
    import traceml_b200 as traceml
    from traceml_b200 import _abi, runtime

    traceml.init(mode="auto")
    eng = runtime.get_engine()
    model = torch.nn.Sequential(torch.nn.Linear(1024, 4096), torch.nn.GELU(), torch.nn.Linear(4096, 1024),
                                torch.nn.LayerNorm(1024), torch.nn.Linear(1024, 16)).cuda()
    traceml.trace_model_instance(model)
    prof = deep.profile_of(model)
    assert prof is not None and len(prof.names) == 5
    x = torch.randn(256, 1024, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            model(x).sum().backward()
    torch.cuda.current_stream().wait_stream(side)
    prof.commit(0)                   # the warm-up's layer calls are not part of the eager step
    torch.cuda.synchronize()
    prof.drain()
    with traceml.trace_step(model):  # one eager step: the activation bytes of these shapes
        model(x).sum().backward()
    torch.cuda.synchronize()
    eager = prof.drain()[-1]
    for p in model.parameters():
        p.grad = None
    # one layer bracketed by events recorded just outside / just inside its region (hooks
    # prepended run before the profile's, hooks appended after)
    evs = tuple(_timed_event() for _ in range(4))
    m0 = model[0]
    hooks = [m0.register_forward_pre_hook(lambda *a: evs[0].record(), prepend=True),
             m0.register_forward_pre_hook(lambda *a: evs[2].record()),
             m0.register_forward_hook(lambda *a: evs[3].record(), prepend=True),
             m0.register_forward_hook(lambda *a: evs[1].record())]
    g = torch.cuda.CUDAGraph()
    with traceml.trace_graph(model):
        with torch.cuda.graph(g):
            model(x).sum().backward()
    for h in hooks:
        h.remove()
    # the graph writes into the current layer accumulators: they cannot be reallocated under it
    assert _lib().tml_layer_init(eng._h, 5, 16) == -3
    torch.cuda.synchronize()
    prof.drain()
    rng = np.random.default_rng(3)
    reps = rng.integers(1, 4, 12)
    for r in reps:
        with traceml.trace_step(model):
            for _ in range(int(r)):
                g.replay()
    torch.cuda.synchronize()
    recs = prof.drain()
    assert recs.shape == (len(reps), 5)
    for k, r in enumerate(reps):
        assert (recs["fwd_calls"][k] == r).all(), (k, r, recs["fwd_calls"][k])
        assert (recs["bwd_calls"][k, 1:] == r).all(), (k, r, recs["bwd_calls"][k])
        assert (recs["fwd_bytes"][k] == r * eager["fwd_bytes"]).all()
        assert (recs["bwd_bytes"][k, 1:] == r * eager["bwd_bytes"][1:]).all()
    assert (recs["fwd_ns"] > 0).all()
    stamp, outer, inner = [], [], []
    for _ in range(16):
        with traceml.trace_step(model):
            g.replay()
        torch.cuda.synchronize()
        outer.append(evs[0].elapsed_time(evs[1]) * 1000.0)
        inner.append(evs[2].elapsed_time(evs[3]) * 1000.0)
        stamp.append(float(prof.drain()[-1]["fwd_ns"][0]) / 1000.0)
    stamp, outer, inner = np.array(stamp), np.array(outer), np.array(inner)
    tol = 2.0 + 0.01 * stamp
    assert (stamp <= outer + tol).all() and (stamp >= inner - tol).all(), (stamp, outer, inner)
    del g
    assert _wait_graph_refs(0) == 0
    assert _lib().tml_layer_init(eng._h, 5, 16) == _abi.TML_OK   # free again once the graph is gone
    deep.reset()


# ------------------------------------------------------------------------------------------- 5
def test_graph_keeps_the_device_state_it_writes_to(cuda):
    from traceml_b200.engine import Engine

    lib = _lib()
    assert _wait_graph_refs(0) == 0
    eng = Engine(device=0, ring_slots=64)
    s = torch.cuda.current_stream().cuda_stream
    assert lib.tml_graph_phase_begin(eng._h, FWD, s) == -3        # not capturing
    x = torch.zeros(1 << 20, device="cuda")

    def body():
        x.add_(1)

    g, _ = _capture_stamped(eng, FWD, body)
    assert lib.tml_graph_refs() == 1
    g.replay()
    assert eng.step_commit(1, 0, 0, 0, 0.0, s) == 0
    torch.cuda.synchronize()
    recs, _ = eng.drain()
    assert len(recs) == 1 and int(recs["n_calls"][0, FWD]) == 1
    assert eng.close() == 1                 # the device state stayed allocated for the graph
    assert lib.tml_graph_refs() == 1        # the graph is never replayed after the close
    del g
    torch.cuda.synchronize()
    gc.collect()
    assert _wait_graph_refs(0) == 0


# ------------------------------------------------------------------------------------------- 6
def test_capture_outside_trace_graph_is_unchanged(cuda):
    from traceml_b200 import _abi
    from traceml_b200.engine import Engine
    from traceml_b200.utils import timing

    lib = _lib()
    eng = Engine(device=0, ring_slots=64)
    refs = lib.tml_graph_refs()
    x = torch.zeros(1 << 20, device="cuda")
    timing._ENG or timing._resolve()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        assert eng.phase_begin(FWD, s) == _abi.TML_ERR_CAPTURE
        assert eng.phase_end(FWD, 0, s) == _abi.TML_ERR_CAPTURE
        r = timing.timed_region("_traceml_internal:forward_time", "step", True)
        with r:
            x.add_(1)
            assert r.slot == _abi.TML_ERR_CAPTURE   # host clock, as before
    assert lib.tml_graph_refs() == refs             # nothing was captured into the graph
    timing._ENG.step_discard()                      # the capture's host-clock region
    del g
    eng.close()
