"""GPU: the live layer-time panel (``live.LayerCombinedTimerData``, csrc/tml_combined.cuh's layer tick)
against the unmodified reference computer fed the same records, against the numpy restatement of its
rules on seeded rings, under CUDA-graph replays, and off the training stream.  Several engines in one
process stand in for ranks.  Every compared value is ``==``."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import layer_tick_cases as ltc  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _model(n_out=8):
    return torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128),
                               torch.nn.LayerNorm(128), torch.nn.Linear(128, n_out)).cuda()


class _Ranks:
    """R engines + layer profiles on cuda:0, closed on exit."""

    def __init__(self, models, ring_steps):
        from traceml_b200.engine import Engine
        from traceml_b200.instrumentation.layers import LayerProfile

        R = len(models)
        self.engines = [Engine(device=0, rank=r, world=R, ring_slots=64, proc_slots=64) for r in range(R)]
        self.profiles = [LayerProfile(e, m, ring_steps=ring_steps) for e, m in zip(self.engines, models)]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        for p in self.profiles:
            p.detach()
        for e in self.engines:
            e.close()


def _load(profile, recs):
    from traceml_b200 import _abi

    recs = np.ascontiguousarray(recs)
    _abi.check(_abi.lib().tml_layer_load_(profile.engine._h, recs.ctypes.data, len(recs), None), "tml_layer_load_")


# ------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize("R", [1, 2, 4, 7])
def test_against_the_reference_computer(cuda, monkeypatch, R):
    if not ltc.reference_importable():
        pytest.skip("reference not installed in oracle/_ref")
    from traceml_b200.live import LayerCombinedTimerData

    torch.manual_seed(R)
    ring = 32
    models = [_model() for _ in range(R)]
    x = torch.randn(32, 64, device="cuda")
    with _Ranks(models, ring) as ranks:
        names = ranks.profiles[0].names
        twin = LayerCombinedTimerData(ranks.profiles, top_n_layers=3)
        ref = ltc.reference_computer(monkeypatch, R, top_n_layers=3)
        drained = {r: [] for r in range(R)}
        step = [0] * R
        ticks = 0
        for tick in range(5):
            for r, (m, p) in enumerate(zip(models, ranks.profiles)):
                for _ in range(6 + (r + tick) % 3):   # ranks end at different steps
                    step[r] += 1
                    m(x).square().mean().backward()
                    p.commit(step[r])
                if tick == 3 and r == 0:              # an eval step: forward rows only
                    step[r] += 1
                    with torch.no_grad():
                        m(x)
                    p.commit(step[r])
            torch.cuda.synchronize()
            for r, p in enumerate(ranks.profiles):
                drained[r].append(p.drain())
            recs = {r: np.concatenate(v)[-ring:] for r, v in drained.items()}
            for _ in range(2):                        # the EMA moves even when the safe step does not
                got = twin.compute_display_data()
                want = ltc.reference_tick(ref, recs, names)
                ltc.assert_same_result(got, want, f"R={R} tick={tick}")
                ticks += 1
        assert got["safe_step"] is not None and got["status_message"] == want["status_message"]
    assert ticks == 10


# ------------------------------------------------------------------------------------------- 2
def _seeded_twin(case, n_layers, top_n=20):
    from traceml_b200.live import LayerCombinedTimerData

    world, recs, ring = ltc.seeded(case, n_layers)
    models = [torch.nn.Sequential(*[torch.nn.Identity() for _ in range(n_layers)]) for _ in range(world)]
    ranks = _Ranks(models, ring)
    for r, p in enumerate(ranks.profiles):
        _load(p, recs[r])
    return ranks, LayerCombinedTimerData(ranks.profiles, top_n_layers=top_n), ltc.retained(recs, ring), world


@pytest.mark.parametrize("case", ltc.SEEDED)
@pytest.mark.parametrize("n_layers", [1, 31, 32, 33, 1024])
def test_seeded_rings(cuda, monkeypatch, case, n_layers):
    ranks, twin, recs, world = _seeded_twin(case, n_layers)
    with ranks:
        names = ranks.profiles[0].names
        got = twin.compute_display_data()
        ltc.check_first_tick(got, ltc.restate(recs, world), names, world)
        if ltc.reference_importable():
            want = ltc.reference_tick(ltc.reference_computer(monkeypatch, world), recs, names)
            ltc.assert_same_result(got, want, case)
    if case == "no_bwd_single":
        assert got["safe_step"] is None and got["missing_ranks"] == [0]
    if case == "no_bwd_rank":
        assert got["safe_step"] == 10 and got["missing_ranks"] == [1]
    if case == "eval_step":
        assert got["safe_step"] == 11
    if case == "ties":
        assert all(r["worst_rank"] == 0 for r in got["all_items"])


@pytest.mark.parametrize("top", ["zero", "one", "all", "more"])
def test_top_n_layers(cuda, top):
    n = 33
    top_n = {"zero": 0, "one": 1, "all": n, "more": n + 7}[top]
    ranks, twin, recs, world = _seeded_twin("staggered", n, top_n=top_n)
    with ranks:
        got = twin.compute_display_data()
    assert len(got["all_items"]) == n and len(got["top_items"]) == min(top_n, n)
    ltc.check_top_n(got, top_n)


# ------------------------------------------------------------------------------------------- 3
@pytest.fixture()
def fresh_deep(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    monkeypatch.setenv("TRACEML_PROFILE", "deep")
    import traceml_b200 as traceml
    from traceml_b200 import runtime
    from traceml_b200.instrumentation import layers
    from traceml_b200.runtime import reset_trace_session_state

    runtime.shutdown_engine()
    reset_trace_session_state(0)
    layers.reset()
    traceml.init(mode="auto")
    yield runtime.get_engine(), layers
    torch.cuda.synchronize()
    layers.reset()
    gc.collect()
    runtime.shutdown_engine()
    reset_trace_session_state(0)


def test_graph_replays(fresh_deep):
    import traceml_b200 as traceml
    from traceml_b200.live import LayerCombinedTimerData

    eng, layers = fresh_deep
    model = _model()
    traceml.trace_model_instance(model)
    prof = layers.profile_of(model)
    x = torch.randn(32, 64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            model(x).sum().backward()
    torch.cuda.current_stream().wait_stream(side)
    prof.commit(0)
    torch.cuda.synchronize()
    with traceml.trace_step(model):
        model(x).sum().backward()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with traceml.trace_graph(model), torch.cuda.graph(g):
        with traceml.trace_step(model):
            model(x).sum().backward()
    torch.cuda.synchronize()
    twin = LayerCombinedTimerData([prof])
    for k in (3, 5):
        for _ in range(k):
            g.replay()
        torch.cuda.synchronize()
        got = twin.compute_display_data()
        steps, _ = eng.drain()
        assert got["safe_step"] == int(steps["step"][-1]), (got["status_message"], steps["step"])
        assert got["missing_ranks"] == [] and len(got["all_items"]) == len(prof.names)
        assert all(r["forward_current"] > 0.0 for r in got["all_items"])
    del g


# ------------------------------------------------------------------------------------------- 4
def test_tick_stays_off_the_training_stream(cuda):
    """The tick neither waits for the training stream nor enqueues on it: with a long kernel queued
    on the training stream, a tick returns while that kernel still runs, and reads the commits that
    completed before it."""
    from traceml_b200.live import LayerCombinedTimerData

    model = _model()
    x = torch.randn(32, 64, device="cuda")
    with _Ranks([model], 16) as ranks:
        p = ranks.profiles[0]
        for s in range(1, 6):
            model(x).sum().backward()
            p.commit(s)
        torch.cuda.synchronize()
        twin = LayerCombinedTimerData([p])
        assert twin.compute_display_data()["safe_step"] == 5  # warm: modules loaded, workspace allocated
        train = torch.cuda.current_stream()
        done = torch.cuda.Event()
        torch.cuda._sleep(1_000_000_000)                      # ~0.5 s of spinning on the training stream
        model(x).sum().backward()
        p.commit(6)                                           # queued behind the spin
        done.record(train)
        got = twin.compute_display_data()
        assert not done.query(), "the tick waited for the training stream"
        assert torch.cuda.current_stream() == train
        assert got["safe_step"] == 5 and got["status_message"] == "Timing snapshot ready."
        done.synchronize()
        assert twin.compute_display_data()["safe_step"] == 6


# ------------------------------------------------------------------------------------------- 5
def test_layer_lists_differ(cuda):
    from traceml_b200.live import LayerCombinedTimerData

    models = [_model(), torch.nn.Sequential(torch.nn.Linear(64, 8), torch.nn.ReLU()).cuda(), _model()]
    x = torch.randn(32, 64, device="cuda")
    with _Ranks(models, 16) as ranks:
        for m, p in zip(models, ranks.profiles):
            m(x).sum().backward()
            p.commit(1)
        torch.cuda.synchronize()
        got = LayerCombinedTimerData(ranks.profiles).compute_display_data()
    assert got["safe_step"] is None and got["all_items"] == [] and got["missing_ranks"] == [0, 1, 2]
    assert "ranks [1]" in got["status_message"]
