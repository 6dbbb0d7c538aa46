"""GPU: steps captured into a CUDA graph (``trace_step`` under ``trace_graph``, tml_graph_step_*)
commit one record per captured step on every replay, under ids the device assigns, with a
device-stamped wall; host steps, host-clock phases and the deep profile interleave with the replays.
The checks are physical (CUDA events recorded inside the same graph) and exact on ids, counts,
memory and the summary sections."""
import gc
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DL, FWD, BWD, OPT, WALL = 0, 2, 3, 4, 5
HAS_MEM = 1


@pytest.fixture()
def fresh(monkeypatch):
    """A new process engine (device-committed mode lasts for an engine's life), closed afterwards."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    import traceml_b200 as traceml
    from traceml_b200 import runtime
    from traceml_b200.runtime import reset_trace_session_state

    runtime.shutdown_engine()
    reset_trace_session_state(0)
    traceml.init(mode="auto")
    yield runtime.get_engine()
    torch.cuda.synchronize()
    gc.collect()
    runtime.shutdown_engine()
    reset_trace_session_state(0)


def _lib():
    from traceml_b200 import _abi

    return _abi.lib()


def _ev():
    return torch.cuda.Event(enable_timing=True, external=True)


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
    return model, opt, x, y


def _train(model, opt, x, y):
    opt.zero_grad(set_to_none=False)
    torch.nn.functional.cross_entropy(model(x), y).backward()
    opt.step()


def _eager_steps(traceml, model, opt, x, y, n, fail_at=()):
    for k in range(n):
        try:
            with traceml.trace_step(model):
                _train(model, opt, x, y)
                if k in fail_at:
                    raise RuntimeError("evaluation failed")
        except RuntimeError:
            pass


def _capture_steps(traceml, model, opt, x, y, k, events=False):
    """A graph of `k` captured steps; with `events`, per step (outer0, outer1, inner0, inner1)
    recorded just outside and just inside its trace_step."""
    g = torch.cuda.CUDAGraph()
    evs = [tuple(_ev() for _ in range(4)) for _ in range(k)] if events else None
    torch.cuda.synchronize()
    with traceml.trace_graph(model), torch.cuda.graph(g):
        for i in range(k):
            if evs:
                evs[i][0].record()
            with traceml.trace_step(model):
                if evs:
                    evs[i][2].record()
                _train(model, opt, x, y)
                if evs:
                    evs[i][3].record()
            if evs:
                evs[i][1].record()
    return g, evs


def _certified_host(recs, window):
    """The host's density check of the retained ring (window_certified's conditions)."""
    n = len(recs)
    steps = recs["step"].astype(np.int64)
    usable = (recs["dur_ns"][:, [0, 2, 3, 4, 5]] > 0).any(axis=1)
    t_start = max(0, n - window)
    return bool((np.diff(steps) == 1).all() and ((recs["flags"] & HAS_MEM) != 0).all() and usable[t_start:].all())


# ------------------------------------------------------------------------------------------- 1
def test_three_steps_captured_in_one_graph(fresh):
    import traceml_b200 as traceml
    from helpers import build_vs_row_oracles
    from traceml_b200.runtime import get_trace_session_state

    eng = fresh
    model, opt, x, y = _graph_model()
    _eager_steps(traceml, model, opt, x, y, 5)
    g, evs = _capture_steps(traceml, model, opt, x, y, 3, events=True)
    assert get_trace_session_state().step == 5          # capturing created no step
    torch.cuda.synchronize()
    mem = (torch.cuda.memory_allocated(), torch.cuda.memory_reserved())
    s = torch.cuda.current_stream()
    n = 40
    torch.cuda._sleep(int(0.1 * 1.9e9))                 # ~0.1 s of device time ahead of the loop
    for _ in range(n):
        g.replay()
    assert not s.query(), "the queued work finished before the loop did: the host was not ahead"
    torch.cuda.synchronize()
    # the brackets: one replay at a time (the graph's events are re-recorded by the next replay)
    m = 8
    outer, inner = [], []
    for _ in range(m):
        g.replay()
        torch.cuda.synchronize()
        outer.append([a.elapsed_time(b) * 1000.0 for a, b, _, _ in evs])
        inner.append([c.elapsed_time(d) * 1000.0 for _, _, c, d in evs])
    recs, dropped = eng.drain()
    assert dropped == 0 and len(recs) == 5 + 3 * (n + m)
    assert list(recs["step"]) == list(range(1, len(recs) + 1))
    assert get_trace_session_state().step == len(recs)
    cap = recs[5:]
    for p in (FWD, BWD, OPT, WALL):
        assert (cap["n_calls"][:, p] == 1).all(), (p, cap["n_calls"][:, p])
        assert (cap["dur_ns"][:, p] > 0).all(), p
    assert (cap["flags"] & HAS_MEM).all()
    assert (cap["peak_alloc"] == mem[0]).all() and (cap["peak_resv"] == mem[1]).all(), (cap["peak_alloc"][:3], mem)
    assert mem == (torch.cuda.memory_allocated(), torch.cuda.memory_reserved())
    tail = cap[-3 * m:]
    outer, inner = np.array(outer).reshape(-1), np.array(inner).reshape(-1)
    wall = tail["dur_ns"][:, WALL].astype(np.float64) / 1000.0
    tol = 2.0 + 0.01 * wall
    hist = {"wall": wall.tolist(), "outer": outer.tolist(), "inner": inner.tolist()}
    assert (wall <= outer + tol).all() and (wall >= inner - tol).all(), hist
    for p in (FWD, BWD, OPT):
        d = tail["dur_ns"][:, p].astype(np.float64) / 1000.0
        assert (d <= inner + 2.0 + 0.01 * d).all(), (p, d.tolist(), inner.tolist())
    compute = tail["dur_ns"][:, [FWD, BWD, OPT]].sum(axis=1).astype(np.float64) / 1000.0
    assert (compute <= inner + 2.0 + 0.01 * compute).all(), (compute.tolist(), inner.tolist())
    assert _lib().tml_ring_certified_(eng._h, len(recs)) == 1
    build_vs_row_oracles(eng, recs, len(recs))
    build_vs_row_oracles(eng, recs, 64)
    del g


# ------------------------------------------------------------------------------------------- 2
def test_host_and_captured_steps_interleave(fresh):
    import traceml_b200 as traceml
    from helpers import build_vs_row_oracles

    eng = fresh
    lib = _lib()
    model, opt, x, y = _graph_model()
    _eager_steps(traceml, model, opt, x, y, 3)
    g, _ = _capture_steps(traceml, model, opt, x, y, 1)
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    assert eng.step_count == 8
    assert lib.tml_ring_certified_(eng._h, 8) == 1
    _eager_steps(traceml, model, opt, x, y, 4, fail_at=(2,))   # completes, completes, raises, completes
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    recs, _ = eng.drain()
    want = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14]
    assert list(recs["step"]) == want
    assert eng.step_count == len(want)
    for w in (1, 3, 4, 5, 8, len(want)):
        assert lib.tml_ring_certified_(eng._h, w) == int(_certified_host(recs, w)), w
    build_vs_row_oracles(eng, recs, len(want))   # no TML_ERR_NONMONOTONIC: the build succeeds
    build_vs_row_oracles(eng, recs, 4)
    del g


# ------------------------------------------------------------------------------------------- 3
class _SleepyData(torch.utils.data.Dataset):
    def __init__(self, n, sleep_s):
        self.n, self.sleep_s = n, sleep_s

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        time.sleep(self.sleep_s)
        return torch.full((4,), float(i))


def test_input_wait_lands_in_the_step_the_next_replay_commits(fresh):
    import traceml_b200 as traceml

    eng = fresh
    model, opt, x, y = _graph_model()
    _eager_steps(traceml, model, opt, x, y, 2)
    g, _ = _capture_steps(traceml, model, opt, x, y, 1)
    torch.cuda.synchronize()
    eng.drain()
    sleep_s, n = 0.02, 8
    loader = torch.utils.data.DataLoader(_SleepyData(n, sleep_s), batch_size=None)
    for _ in loader:
        g.replay()
    torch.cuda.synchronize()
    recs, _ = eng.drain()
    assert list(recs["step"]) == list(range(3, 3 + n))
    dl_ms = recs["dur_ns"][:, DL].astype(np.float64) / 1.0e6
    assert (recs["n_calls"][:, DL] == 1).all(), recs["n_calls"][:, DL]
    assert (dl_ms >= sleep_s * 1000.0 * 0.95).all() and (dl_ms < sleep_s * 1000.0 + 30.0).all(), dl_ms.tolist()
    del g


# ------------------------------------------------------------------------------------------- 4
@pytest.fixture()
def deep(monkeypatch, fresh):
    monkeypatch.setenv("TRACEML_PROFILE", "deep")
    from traceml_b200.instrumentation import layers

    layers.reset()
    yield layers
    layers.reset()


def test_deep_profile_in_captured_steps(fresh, deep):
    import traceml_b200 as traceml

    eng = fresh
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
    prof.commit(0)                   # the warm-up's layer calls are not part of an eager step
    torch.cuda.synchronize()
    for _ in range(2):               # eager steps 1, 2
        with traceml.trace_step(model):
            model(x).sum().backward()
    for p in model.parameters():
        p.grad = None
    evs = tuple(_ev() for _ in range(4))
    m0 = model[0]
    hooks = [m0.register_forward_pre_hook(lambda *a: evs[0].record(), prepend=True),
             m0.register_forward_pre_hook(lambda *a: evs[2].record()),
             m0.register_forward_hook(lambda *a: evs[3].record(), prepend=True),
             m0.register_forward_hook(lambda *a: evs[1].record())]
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with traceml.trace_graph(model), torch.cuda.graph(g):
        with traceml.trace_step(model):
            model(x).sum().backward()
    for h in hooks:
        h.remove()
    torch.cuda.synchronize()
    prof.drain()
    eng.drain()
    stamp, outer, inner = [], [], []
    n = 12
    for _ in range(n):
        g.replay()
        torch.cuda.synchronize()
        outer.append(evs[0].elapsed_time(evs[1]) * 1000.0)
        inner.append(evs[2].elapsed_time(evs[3]) * 1000.0)
        stamp.append(float(prof.drain()[-1]["fwd_ns"][0]) / 1000.0)
    torch.cuda.synchronize()
    steps, _ = eng.drain()
    assert list(steps["step"]) == list(range(3, 3 + n))
    with traceml.trace_step(model):   # a host step after the replays: the device's next id
        model(x).sum().backward()
    torch.cuda.synchronize()
    last = prof.drain()
    assert last.shape == (1, 5) and (last["step"] == 3 + n).all()
    stamp, outer, inner = np.array(stamp), np.array(outer), np.array(inner)
    tol = 2.0 + 0.01 * stamp
    assert (stamp <= outer + tol).all() and (stamp >= inner - tol).all(), (stamp, outer, inner)
    # one record per replayed step, under the device's ids (checked one replay at a time above;
    # here: a burst of replays drained at once)
    for _ in range(4):
        g.replay()
    torch.cuda.synchronize()
    recs = prof.drain()
    assert recs.shape == (4, 5)
    assert [int(r[0]) for r in recs["step"]] == list(range(4 + n, 8 + n))
    assert (recs["fwd_calls"] == 1).all() and (recs["bwd_calls"][:, 1:] == 1).all()
    del g


# ------------------------------------------------------------------------------------------- 5
def test_graph_with_a_captured_commit_keeps_the_device_state(fresh):
    from traceml_b200.engine import Engine

    lib = _lib()
    eng = Engine(device=0, ring_slots=64)
    s = torch.cuda.current_stream().cuda_stream
    assert lib.tml_graph_step_begin(eng._h, s) == -3           # not capturing
    x = torch.zeros(1 << 20, device="cuda")
    torch.cuda.synchronize()
    refs = int(lib.tml_graph_refs())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream().cuda_stream
        slot = lib.tml_graph_step_begin(eng._h, cs)
        assert slot == 0, slot
        x.add_(1)
        assert lib.tml_graph_step_commit(eng._h, 0, cs) == 0
    assert lib.tml_graph_refs() == refs + 1
    assert lib.tml_graph_step_publish(eng._h, 41, 0, 0, s) == 0   # the id before any commit: 41
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    recs, _ = eng.drain()
    assert list(recs["step"]) == [42, 43] and (recs["n_calls"][:, WALL] == 1).all()
    assert eng.graph_step_id() == 43 and eng.step_count == 2
    assert eng.close() == 1                 # the device state stayed allocated for the graph
    assert lib.tml_graph_refs() == refs + 1
    del g
    torch.cuda.synchronize()
    gc.collect()
    t0 = time.monotonic()
    while lib.tml_graph_refs() != refs and time.monotonic() - t0 < 10.0:
        gc.collect()
        time.sleep(0.01)
    assert lib.tml_graph_refs() == refs


# ------------------------------------------------------------------------------------------- 6
def test_two_contexts_as_two_ranks(fresh):
    """Each context captures its own step; rank 1 replays more often.  The multi-rank sections
    (the Python-sequenced driver) equal the row oracles."""
    import replay
    from helpers import assert_struct, oracle_mem_rows, oracle_time_rows, plain, strip_device
    from oracle import step_memory_oracle, step_time_oracle
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    lib = _lib()
    R = 2
    engines = [Engine(device=0, rank=r, world=R, ring_slots=256) for r in range(R)]
    s = torch.cuda.current_stream().cuda_stream
    mats = [torch.randn(512, 512, device="cuda") for _ in range(R)]
    torch.cuda.synchronize()
    graphs = []
    for r, e in enumerate(engines):
        for k in range(3):                  # eager steps 1..3
            slot = e.phase_begin(FWD, s)
            mats[r] @ mats[r]
            assert e.phase_end(FWD, slot, s) == 0
            assert e.step_commit(k + 1, 1000 + r, 2000 + r, HAS_MEM, 0.0, s) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cs = torch.cuda.current_stream().cuda_stream
            assert lib.tml_graph_step_begin(e._h, cs) == 0
            gs = lib.tml_graph_phase_begin(e._h, FWD, cs)
            assert gs == 1
            mats[r] @ mats[r]
            assert lib.tml_graph_phase_end(e._h, FWD, gs, cs) == 0
            assert lib.tml_graph_step_commit(e._h, HAS_MEM, cs) == 0
        assert lib.tml_graph_step_publish(e._h, 0, 5000 + r, 6000 + r, s) == 0
        graphs.append(g)
    for r, g in enumerate(graphs):
        for _ in range(10 + 7 * r):
            g.replay()
    torch.cuda.synchronize()
    recs = {}
    for r, e in enumerate(engines):
        recs[r], _ = e.drain()
        assert list(recs[r]["step"]) == list(range(1, 14 + 7 * r))
        assert (recs[r]["peak_alloc"][3:] == 5000 + r).all()
    W = 12
    try:
        got = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R).build(W, W)
        o = step_time_oracle.step_time_section(oracle_time_rows(recs, W), max_rows=W)
        gt = got["step_time"]
        assert_struct(plain(gt["data"]), plain({k: o["data"][k] for k in gt["data"]}), "data")
        assert_struct(plain(gt["diagnosis"]), plain(o["diagnosis"]), "diagnosis")
        mo = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=W,
                                                    gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
        gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
        assert_struct(gd["primary"], od["primary"], "mem.primary")
        assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")
    finally:
        del graphs, g
        torch.cuda.synchronize()
        gc.collect()
        for e in engines:
            e.close()
