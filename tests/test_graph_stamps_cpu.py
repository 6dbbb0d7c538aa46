"""CPU: the graph-captured region entry points reject bad arguments without a GPU, and the
timed_region seam routes a capturing stream's regions to them only inside ``trace_graph``
(a fake engine stands in for the native context)."""
import pytest

from traceml_b200 import _abi

TML_ERR_ARG, TML_ERR_STATE = -2, -3


def test_graph_symbols_reject_null_and_bad_arguments_without_a_gpu():
    lib = _abi.lib()
    assert lib.tml_graph_phase_begin(None, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_phase_begin(None, 8, None) == TML_ERR_ARG
    assert lib.tml_graph_phase_end(None, 0, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_phase_end(None, 0, -1, None) == TML_ERR_ARG
    assert lib.tml_graph_layer_begin(None, None) == TML_ERR_ARG
    assert lib.tml_graph_layer_end(None, 0, 0, 0, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_refs() == 0          # no context ever captured a stamp in this process
    assert lib.tml_phase_begin(None, 0, None) == TML_ERR_ARG


class _FakeEngine:
    """The four step-path entry points and the two graph ones, recording what they were asked."""

    def __init__(self, begin_status=_abi.TML_ERR_CAPTURE, graph_status=None):
        self._h = object()
        self.begin_status, self.graph_status = begin_status, graph_status
        self.calls, self.depth = [], 0

    def _begin(self, h, phase, stream):
        self.calls.append(("begin", phase))
        return self.begin_status

    def _end(self, h, phase, slot, stream):
        self.calls.append(("end", phase, slot))
        return 0

    def _host(self, h, phase, dur_ns):
        self.calls.append(("host", phase))
        return 0

    def _gbegin(self, h, phase, stream):
        if self.graph_status is not None:
            self.calls.append(("gbegin_failed", phase))
            return self.graph_status
        slot, self.depth = self.depth, self.depth + 1
        self.calls.append(("gbegin", phase, slot))
        return slot

    def _gend(self, h, phase, slot, stream):
        assert slot == self.depth - 1, "graph regions close LIFO"
        self.depth -= 1
        self.calls.append(("gend", phase, slot))
        return 0


class _FakeFast:
    """traceml_b200._tml_step bound to a fake engine."""

    def __init__(self, eng):
        self.eng = eng

    def begin(self, phase):
        return self.eng._begin(self.eng._h, phase, 0)

    def end(self, phase, slot):
        return self.eng._end(self.eng._h, phase, slot, 0)

    def host(self, phase, dur_ns):
        return self.eng._host(self.eng._h, phase, dur_ns)


@pytest.fixture(params=["ctypes", "native_glue"])
def seam(request, monkeypatch):
    from traceml_b200.instrumentation import patches
    from traceml_b200.utils import timing

    def install(eng):
        monkeypatch.setattr(timing, "_ENG", eng)
        monkeypatch.setattr(timing, "_FAST", _FakeFast(eng) if request.param == "native_glue" else None)
        return eng

    monkeypatch.setattr(timing, "_raw_stream", lambda dev: 0)
    monkeypatch.setattr(timing, "_cur_dev", lambda: 0)
    monkeypatch.setattr(patches, "ensure_optimizer_timing_installed", lambda: None)
    yield install
    assert timing.GRAPH_SCOPE.depth == 0 and timing.GRAPH_SCOPES_OPEN[0] == 0


def _region(name="_traceml_internal:forward_time"):
    from traceml_b200.utils.timing import timed_region

    return timed_region(name, "step", True)


def test_capture_inside_trace_graph_goes_to_the_graph_calls(seam):
    from traceml_b200.sdk import trace_graph

    eng = seam(_FakeEngine())
    with trace_graph():
        with _region():
            pass
    assert eng.calls == [("begin", 2), ("gbegin", 2, 0), ("gend", 2, 0)]


def test_capture_outside_trace_graph_takes_the_host_clock(seam):
    eng = seam(_FakeEngine())
    with _region():
        pass
    assert eng.calls == [("begin", 2), ("host", 2)]


def test_failing_graph_begin_takes_the_host_clock(seam):
    from traceml_b200.sdk import trace_graph

    eng = seam(_FakeEngine(graph_status=TML_ERR_STATE))
    with trace_graph():
        with _region():
            pass
    assert eng.calls == [("begin", 2), ("gbegin_failed", 2), ("host", 2)]


def test_other_begin_failures_inside_trace_graph_take_the_host_clock(seam):
    from traceml_b200.sdk import trace_graph

    eng = seam(_FakeEngine(begin_status=-1))  # TML_ERR_CUDA: not a capture
    with trace_graph():
        with _region():
            pass
    assert eng.calls == [("begin", 2), ("host", 2)]


def test_plain_regions_inside_trace_graph_are_unchanged(seam):
    from traceml_b200.sdk import trace_graph

    eng = seam(_FakeEngine(begin_status=5))
    with trace_graph():
        with _region():
            pass
    assert eng.calls == [("begin", 2), ("end", 2, 5)]


def test_nested_graph_regions_get_slots_by_depth_and_close_lifo(seam):
    from traceml_b200.sdk import trace_graph
    from traceml_b200.utils.timing import GRAPH_SLOT0

    eng = seam(_FakeEngine())
    with trace_graph():
        with _region("_traceml_internal:forward_time") as a:
            with _region("_traceml_internal:backward_time") as b:
                with _region("_traceml_internal:optimizer_step") as c:
                    assert [GRAPH_SLOT0 - r.slot for r in (a, b, c)] == [0, 1, 2]
        with _region("_traceml_internal:forward_time") as d:   # the slot is free again
            assert GRAPH_SLOT0 - d.slot == 0
    assert [x for x in eng.calls if x[0] in ("gbegin", "gend")] == [
        ("gbegin", 2, 0), ("gbegin", 3, 1), ("gbegin", 4, 2),
        ("gend", 4, 2), ("gend", 3, 1), ("gend", 2, 0),
        ("gbegin", 2, 0), ("gend", 2, 0)]
    assert eng.depth == 0


def test_trace_graph_restores_the_opener_flags_when_the_body_raises(seam):
    import torch.nn as nn

    from traceml_b200.instrumentation import patches
    from traceml_b200.sdk import trace_graph
    from traceml_b200.utils import timing

    seam(_FakeEngine())
    model = nn.Linear(2, 2)
    t = patches._TLS
    before = (t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.h2d)
    with pytest.raises(ValueError, match="boom"):
        with trace_graph(model):
            assert t.fwd and t.bwd and t.h2d and t.fwd_targets == frozenset({id(model)})
            assert timing.GRAPH_SCOPE.depth == 1 and timing.GRAPH_SCOPES_OPEN[0] == 1
            raise ValueError("boom")
    assert (t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.h2d) == before
    assert timing.GRAPH_SCOPE.depth == 0 and timing.GRAPH_SCOPES_OPEN[0] == 0


def test_trace_graph_starts_the_engine_before_the_capture(seam, monkeypatch):
    """The engine's creation allocates device memory, which a capture forbids: trace_graph
    creates it on entry, not the first region inside the graph."""
    from traceml_b200.sdk import trace_graph
    from traceml_b200.utils import timing

    eng = _FakeEngine()
    monkeypatch.setattr(timing, "_ENG", None)
    monkeypatch.setattr(timing, "_FAST", None)
    started = []

    def resolve():
        started.append(True)
        timing._ENG = eng
        return eng

    monkeypatch.setattr(timing, "_resolve", resolve)
    with trace_graph():
        assert started == [True]
        with _region():
            pass
    assert started == [True]
    assert eng.calls == [("begin", 2), ("gbegin", 2, 0), ("gend", 2, 0)]


def test_trace_graph_is_public():
    import traceml_b200 as traceml
    from traceml_b200 import sdk

    assert traceml.trace_graph is sdk.trace_graph
    assert "trace_graph" in traceml.__all__
