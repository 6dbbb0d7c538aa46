"""CPU: the graph-captured step entry points reject bad arguments without a GPU, and ``trace_step``
routes a capturing stream's step to them only inside ``trace_graph``; after the first captured
commit, host steps send "advanced or not" and host-clock regions go to the device (a fake engine
stands in for the native context)."""
import ctypes as C

import pytest

from traceml_b200 import _abi

TML_ERR_ARG, TML_ERR_STATE = -2, -3
HAS_MEM = 1


def test_graph_step_symbols_reject_null_and_bad_arguments_without_a_gpu():
    lib = _abi.lib()
    out = C.c_uint64(0)
    assert lib.tml_graph_step_begin(None, None) == TML_ERR_ARG
    assert lib.tml_graph_step_commit(None, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_step_commit(None, HAS_MEM | _abi.TML_GRAPH_STEP_FAILED, None) == TML_ERR_ARG
    assert lib.tml_graph_step_commit(None, 2, None) == TML_ERR_ARG   # not a commit flag
    assert lib.tml_graph_step_publish(None, 0, 0, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_step_id(None, C.byref(out)) == TML_ERR_ARG
    assert lib.tml_graph_phase_host(None, 0, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_phase_host(None, 8, 0, None) == TML_ERR_ARG
    assert lib.tml_graph_layer_commit(None, None) == TML_ERR_ARG
    assert lib.tml_step_count(None) == 0


def test_records_of_captured_steps_match_their_ctypes_mirrors():
    lib = _abi.lib()
    for name, cls in (("tml_step_record", _abi.StepRecord), ("tml_layer_record", _abi.LayerRecord)):
        assert int(lib.tml_struct_size(name.encode())) == C.sizeof(cls), name


class _FakeEngine:
    """The step-path entry points, the graph region ones and the graph step ones, recording what
    they were asked."""

    device = 0

    def __init__(self, begin_status=_abi.TML_ERR_CAPTURE, commit_status=_abi.TML_ERR_CAPTURE):
        self._h = object()
        self.begin_status, self.commit_status = begin_status, commit_status
        self.calls, self.depth, self.dev_step = [], 0, 7

    def _begin(self, h, phase, stream):
        self.calls.append(("begin", phase))
        return self.begin_status

    def _end(self, h, phase, slot, stream):
        self.calls.append(("end", phase, slot))
        return 0

    def _host(self, h, phase, dur_ns):
        self.calls.append(("host", phase))
        return 0

    def _commit(self, h, step, alloc, resv, flags, ts, stream):
        self.calls.append(("commit", step))
        return self.commit_status

    def step_discard(self):
        self.calls.append(("discard",))

    def _gbegin(self, h, phase, stream):
        slot, self.depth = self.depth, self.depth + 1
        self.calls.append(("gbegin", phase, slot))
        return slot

    def _gend(self, h, phase, slot, stream):
        assert slot == self.depth - 1, "graph regions close LIFO"
        self.depth -= 1
        self.calls.append(("gend", phase, slot))
        return 0

    def _gsbegin(self, h, stream):
        slot, self.depth = self.depth, self.depth + 1
        self.calls.append(("gsbegin", slot))
        return slot

    def _gscommit(self, h, flags, stream):
        assert self.depth > 0
        self.depth -= 1
        self.calls.append(("gscommit", flags))
        return 0

    def _gpublish(self, h, base, alloc, resv, stream):
        self.calls.append(("publish", base))
        return 0

    def _ghost(self, h, phase, dur_ns, stream):
        self.calls.append(("ghost", phase))
        return 0

    def graph_step_id(self):
        self.calls.append(("step_id",))
        return self.dev_step


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

    def commit(self, step, mem_dev, ts):
        return self.eng._commit(self.eng._h, step, 0, 0, 0, ts, 0)

    def current_bytes(self, dev):
        return 0, 0

    def reset_peaks(self, dev):
        pass


@pytest.fixture(params=["ctypes", "native_glue"])
def seam(request, monkeypatch):
    from traceml_b200.instrumentation import patches
    from traceml_b200.runtime import get_trace_session_state, reset_trace_session_state
    from traceml_b200.sdk import instrumentation
    from traceml_b200.utils import timing

    capturing = [True]

    def install(eng):
        monkeypatch.setattr(timing, "_ENG", eng)
        monkeypatch.setattr(timing, "_FAST", _FakeFast(eng) if request.param == "native_glue" else None)
        return eng

    monkeypatch.setattr(timing, "_raw_stream", lambda dev: 0)
    monkeypatch.setattr(timing, "_cur_dev", lambda: 0)
    monkeypatch.setattr(timing, "DEVICE_STEPS", False)
    monkeypatch.setattr(patches, "ensure_optimizer_timing_installed", lambda: None)
    monkeypatch.setattr(instrumentation, "_capturing", lambda: capturing[0])
    reset_trace_session_state(3)
    install.capturing = capturing
    yield install
    get_trace_session_state().bind_device_step(None)
    reset_trace_session_state(0)
    assert timing.GRAPH_SCOPE.depth == 0 and timing.GRAPH_SCOPES_OPEN[0] == 0


def _model():
    import torch.nn as nn

    return nn.Linear(2, 2)   # on the CPU: its steps carry no memory


def test_captured_step_inside_trace_graph_goes_to_the_graph_step_calls(seam):
    from traceml_b200.runtime import get_trace_session_state
    from traceml_b200.sdk import trace_graph, trace_step
    from traceml_b200.utils.timing import timed_region

    eng = seam(_FakeEngine())
    model = _model()
    with trace_graph(model):
        for _ in range(2):   # two steps captured in one graph
            with trace_step(model):
                with timed_region("_traceml_internal:forward_time", "step", True):
                    pass
    assert eng.calls == [("gsbegin", 0), ("begin", 2), ("gbegin", 2, 1), ("gend", 2, 1), ("gscommit", 0),
                         ("gsbegin", 0), ("begin", 2), ("gbegin", 2, 1), ("gend", 2, 1), ("gscommit", 0),
                         ("publish", 3)]
    assert eng.depth == 0
    # capturing advanced nothing on the host; the step id is the device's from now on
    assert get_trace_session_state().step == 7


def test_capture_outside_trace_graph_takes_todays_path(seam):
    from traceml_b200.sdk import trace_step
    from traceml_b200.utils import timing

    eng = seam(_FakeEngine())
    with trace_step(_model()):
        pass
    assert not any(c[0] in ("gsbegin", "gscommit", "publish") for c in eng.calls), eng.calls
    assert ("commit", 4) in eng.calls and ("discard",) in eng.calls   # refused under capture, as before
    assert not timing.DEVICE_STEPS


def test_failing_body_inside_a_captured_step_restores_the_opener_flags(seam):
    from traceml_b200.instrumentation import patches
    from traceml_b200.sdk import trace_graph, trace_step
    from traceml_b200.utils import timing

    eng = seam(_FakeEngine())
    model = _model()
    t = patches._TLS
    with trace_graph(model):
        armed = (t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.bwd_depth, t.h2d)
        with pytest.raises(ValueError, match="boom"):
            with trace_step(model):
                assert t.fwd and t.bwd and t.h2d
                t.fwd_depth, t.bwd_depth = 2, 1   # the body was inside a forward / backward
                raise ValueError("boom")
        assert (t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.bwd_depth, t.h2d) == armed
    # the step is committed under the old id, as a failed host step flushes
    assert ("gscommit", _abi.TML_GRAPH_STEP_FAILED) in eng.calls
    assert eng.depth == 0 and timing.GRAPH_SCOPE.depth == 0


def test_failing_graph_step_begin_takes_todays_path(seam, monkeypatch):
    from traceml_b200.sdk import trace_graph, trace_step

    eng = seam(_FakeEngine())
    monkeypatch.setattr(eng, "_gsbegin", lambda h, s: TML_ERR_STATE)
    with trace_graph(_model()):
        with trace_step(_model()):
            pass
    assert not any(c[0] in ("gscommit", "publish") for c in eng.calls), eng.calls
    assert ("discard",) in eng.calls


def test_host_steps_after_a_captured_commit_send_advanced_or_not(seam):
    from traceml_b200.sdk import trace_graph, trace_step
    from traceml_b200.utils.timing import timed_region

    eng = seam(_FakeEngine(commit_status=0))
    model = _model()
    with trace_graph(model):
        with trace_step(model):
            pass
    seam.capturing[0] = False
    eng.calls.clear()
    with trace_step(model):                                    # completes: advanced
        with timed_region("_traceml_internal:dataloader_next", "step", False):
            pass
    with pytest.raises(RuntimeError):
        with trace_step(model):                                # raises: the old id again
            raise RuntimeError("eval failed")
    with timed_region("_traceml_internal:dataloader_next", "step", False):  # between replays
        pass
    # (without the native glue the step's own host-clock region goes to the device too: phase 5)
    assert [c for c in eng.calls if c[0] in ("commit", "publish") or c == ("ghost", 0)] == [
        ("ghost", 0), ("commit", 1), ("publish", 0), ("commit", 0), ("publish", 0), ("ghost", 0)]
    assert ("host", 0) not in eng.calls


def test_regions_before_any_captured_commit_are_unchanged(seam):
    from traceml_b200.utils.timing import timed_region

    eng = seam(_FakeEngine())
    seam.capturing[0] = False
    with timed_region("_traceml_internal:dataloader_next", "step", False):
        pass
    assert eng.calls == [("host", 0)]
