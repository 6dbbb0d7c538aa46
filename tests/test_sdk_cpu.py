"""CPU: SDK policy and host-side semantics (mirrors the intent of the reference's
tests/sdk/test_init_and_wrappers.py:34-417 and tests/runtime/test_trace_session_state.py)."""
import os

import pytest
import torch
import torch.nn as nn

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


@pytest.fixture()
def fresh(monkeypatch):
    from traceml_b200.sdk import initial

    initial._reset_for_tests()
    monkeypatch.setattr(initial, "_require_engine", lambda: None)
    yield initial
    initial._reset_for_tests()


def test_init_policy_matrix(fresh):
    b = fresh._build
    assert b("auto", {}, "u") == fresh.TraceMLInitConfig("auto", True, True, True, True, "u")
    assert b("manual", {}, "u") == fresh.TraceMLInitConfig("manual", False, False, False, False, "u")
    assert b("custom", {"patch_forward": True}, "u").mode == "selective"
    with pytest.raises(ValueError):
        b("turbo", {}, "u")
    with pytest.raises(ValueError):
        b("auto", {"patch_forward": True}, "u")
    with pytest.raises(ValueError):
        b("selective", {}, "u")
    with pytest.raises(ValueError):
        b("selective", {"patch_forward": False}, "u")


def test_init_idempotent_and_conflict(fresh):
    c1 = fresh.init(mode="manual")
    assert fresh.init(mode="manual") is c1
    with pytest.raises(RuntimeError, match="already been initialized"):
        fresh.init(mode="selective", patch_h2d=True)


def test_phase_mapping_follows_reference_buckets():
    from traceml_b200.utils.timing import phase_of

    assert [phase_of(f"_traceml_internal:{n}") for n in
            ("dataloader_next", "h2d_time", "forward_time", "backward_time", "optimizer_step", "step_time")] \
        == [0, 1, 2, 3, 4, 5]
    assert phase_of("my_batch_loader") == 0 and phase_of("fwd") == 2 and phase_of("bwd_pass") == 3
    assert phase_of("update") == 4 and phase_of("checkpoint") == 6


def test_step_state_semantics():
    from traceml_b200.runtime.state import TraceSessionState

    s = TraceSessionState()
    assert s.step == 0 and s.advance_step() == 1 and s.advance_step(2) == 3
    with pytest.raises(ValueError):
        s.set_step(-1)
    with pytest.raises(TypeError):
        s.advance_step(1.5)
    assert s.reset() == 0


def test_should_time_h2d_rules():
    from traceml_b200.instrumentation.h2d import should_time_h2d

    x = torch.zeros(2)
    assert should_time_h2d(x, ("cuda",), {})
    assert should_time_h2d(x, (), {"device": torch.device("cuda", 0)})
    assert not should_time_h2d(x, ("cpu",), {})
    assert not should_time_h2d(x, (torch.float16,), {})
    assert not should_time_h2d(nn.Parameter(x), ("cuda",), {})


def test_wrappers_refuse_to_stack_on_auto_patches(monkeypatch):
    from traceml_b200.sdk import wrappers

    monkeypatch.setattr(nn.Module, "_traceml_forward_patched", True, raising=False)
    with pytest.raises(RuntimeError, match="automatic instrumentation is already active"):
        wrappers.wrap_forward(nn.Linear(2, 2))
    monkeypatch.setattr(nn.Module, "_traceml_forward_patched", False, raising=False)
    with pytest.raises(TypeError):
        wrappers.wrap_forward(object())
    with pytest.raises(TypeError):
        wrappers.wrap_h2d(3)
    with pytest.raises(TypeError):
        wrappers.wrap_dataloader_fetch(3)


def test_disabled_short_circuits_everything(monkeypatch):
    from traceml_b200 import runtime

    monkeypatch.setenv("TRACEML_DISABLED", "1")
    runtime.refresh_disabled()
    try:
        from traceml_b200.sdk.instrumentation import trace_step
        from traceml_b200.utils.timing import timed_region

        ran = []
        with trace_step(nn.Linear(2, 2)):
            with timed_region("_traceml_internal:forward_time"):
                ran.append(1)
        assert ran == [1]
    finally:
        monkeypatch.delenv("TRACEML_DISABLED")
        runtime.refresh_disabled()


def test_forward_targets_include_ddp_and_fsdp_inner():
    from traceml_b200.instrumentation.patches import forward_targets

    inner = nn.Linear(2, 2)

    class Wrap(nn.Module):
        def __init__(self):
            super().__init__()
            self.module = inner

    w = Wrap()
    assert forward_targets(w) == frozenset({id(w), id(inner)})
    assert forward_targets(None) == frozenset()


def test_wire_rows_from_records_match_reference_schema():
    import replay
    from traceml_b200.records import step_record_to_memory_wire, step_record_to_wire

    r = replay.make_step_replay("balanced", 1, 3, seed=0)[0][1]
    w = step_record_to_wire(r, device="cuda:3")
    assert set(w) == {"seq", "timestamp", "step", "events"} and w["step"] == 2
    ev = w["events"]["_traceml_internal:forward_time"]["cuda:3"]
    assert ev["is_gpu"] is True and ev["n_calls"] == 1 and ev["duration_ms"] == int(r["dur_ns"][2]) / 1e6
    assert "cpu" in w["events"]["_traceml_internal:step_time"]
    m = step_record_to_memory_wire(r, device="cuda:3")
    assert set(m) == {"seq", "ts", "model_id", "device", "step", "peak_alloc", "peak_resv"}
    assert m["peak_alloc"] == float(int(r["peak_alloc"]))


def test_kept_huggingface_integration_imports_against_this_package(monkeypatch):
    """The kept ``integrations/huggingface.py`` with its single TraceML import line pointed at
    this package: it must import (TRACEML_DISABLED: no engine needed), expose ``TraceMLTrainer``
    on top of transformers' Trainer, and its bypass path must not touch the engine."""
    import importlib.util
    import sys
    import types

    ref = os.path.join(REF, "traceml", "integrations", "huggingface.py")
    if not os.path.exists(ref):
        pytest.skip("the reference is not installed in oracle/_ref")
    pytest.importorskip("transformers")
    monkeypatch.setenv("TRACEML_DISABLED", "1")
    from traceml_b200 import runtime

    runtime.refresh_disabled()
    try:
        src = open(ref).read()
        line = "from traceml.sdk.decorators_compat import trace_model_instance, trace_step"
        assert src.count(line) == 1
        src = src.replace(line, "from traceml_b200.sdk.decorators_compat import trace_model_instance, trace_step")
        assert "traceml." not in src.replace("traceml_b200.", "")  # nothing else of TraceML is imported
        mod = types.ModuleType("kept_hf_integration")
        exec(compile(src, ref, "exec"), mod.__dict__)
        from transformers import Trainer

        assert issubclass(mod.TraceMLTrainer, Trainer) and mod.TRACEML_DISABLED is True
        import traceml_b200.sdk.decorators_compat as compat

        assert compat.trace_step is mod.trace_step
    finally:
        monkeypatch.delenv("TRACEML_DISABLED")
        runtime.refresh_disabled()


def test_kept_lightning_callback_imports_against_this_package(monkeypatch):
    """The kept ``integrations/lightning.py`` with its TraceML imports pointed at this package's
    seam modules (same module paths, same names): it must import and define its callback.
    (Lightning itself is stubbed: only ``Callback`` is needed at import time; the hook sequence
    is exercised on the GPU by test_gpu_step_path.py::test_lightning_style_seam_sequence.)"""
    import sys
    import types

    ref = os.path.join(REF, "traceml", "integrations", "lightning.py")
    if not os.path.exists(ref):
        pytest.skip("the reference is not installed in oracle/_ref")
    src = open(ref).read()
    wanted = ["from traceml.runtime.state import", "from traceml.utils.flush_buffers import",
              "from traceml.utils.step_memory import", "from traceml.utils.timing import"]
    for w in wanted:
        assert src.count(w) == 1, w
    src = src.replace("from traceml.", "from traceml_b200.")
    for name in ("lightning", "lightning.pytorch", "lightning.pytorch.callbacks"):
        monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
    sys.modules["lightning.pytorch.callbacks"].Callback = type("Callback", (), {})
    mod = types.ModuleType("kept_lightning_integration")
    exec(compile(src, ref, "exec"), mod.__dict__)
    cbs = [v for v in vars(mod).values() if isinstance(v, type) and v.__module__ == mod.__name__
           and issubclass(v, sys.modules["lightning.pytorch.callbacks"].Callback)]
    assert cbs, "the kept file defines its Lightning callback"
    for name in ("get_trace_session_state", "flush_step_events", "StepMemoryTracker", "TimeEvent",
                 "TimeScope", "record_event", "timed_region"):
        assert getattr(mod, name).__module__.startswith("traceml_b200."), name
