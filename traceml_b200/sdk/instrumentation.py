"""``trace_step`` (mirror of ``src/traceml/sdk/instrumentation.py:160-200``).

Step boundary semantics kept exactly: reset allocator peaks; open the
host-clock ``step_time`` region; raise the auto-timer flags; install optimizer
hooks on first use in auto mode; on exit advance the step counter only if the
body completed, record peaks, and flush under the (possibly advanced) step id
-- a failed step therefore flushes under the old id.  Telemetry never raises;
user exceptions propagate.

A ``trace_step`` entered on a capturing stream inside ``trace_graph`` is a
captured step: its begin stamp and its commit go into the graph, and every
replay commits one step record with a device-stamped ``step_time`` under the id
the device assigns.  From the first captured commit on, the engine counts steps
on the device (device-committed mode): host steps send only "advanced or not",
and host-clock phases are added on the device.
"""
from __future__ import annotations

import functools
import os
import sys
import time
from typing import Callable

from .._abi import TML_GRAPH_STEP_FAILED
from ..instrumentation import patches as _patches
from ..records import FLAG_HAS_MEM, PHASE_STEP
from ..runtime import disabled, get_trace_session_state
from ..utils import timing as _timing
from ..utils.flush_buffers import flush_step_events
from ..utils.step_memory import StepMemoryTracker
from ..utils.timing import timed_region
from . import initial as _initial

STEP = "_traceml_internal:step_time"
_perf_ns = time.perf_counter_ns
_wall = time.time
_STATE = get_trace_session_state()
_INFO_KEY = "_traceml_b200_info"
_INFO_TTL = 256  # steps between re-checks of the model's device


def _auto_optimizer() -> bool:
    cfg = _initial._CONFIG
    return cfg is None or cfg.mode == "auto"


def _model_info(model):
    """(mem_device or -1, forward target ids, ttl) cached on the model instance: the
    device lookup and the DDP/FSDP unwrapping are not redone every step."""
    info = model.__dict__.get(_INFO_KEY)
    if info is not None and info[2][0] > 0:
        info[2][0] -= 1
        return info
    tracker = StepMemoryTracker(model)
    info = (tracker.index if tracker.is_cuda else -1, _patches.forward_targets(model), [_INFO_TTL])
    try:
        model.__dict__[_INFO_KEY] = info
    except Exception:
        pass
    return info


def _log(message: str, exc: Exception) -> None:
    print(f"[TraceML] {message}: {exc}", file=sys.stderr)


def _capturing() -> bool:
    import torch

    return torch.cuda.is_current_stream_capturing()


def _publish(eng, mem_dev: int, base_step: int = 0) -> None:
    """Device-committed mode: the allocator's current bytes for the captured commits that follow
    (outside any capture: at trace_graph exit and after every host commit)."""
    import torch

    alloc = resv = 0
    if mem_dev >= 0:
        fast = _timing._FAST
        alloc, resv = (fast.current_bytes(mem_dev) if fast is not None
                       else (torch.cuda.memory_allocated(mem_dev), torch.cuda.memory_reserved(mem_dev)))
    rc = eng._gpublish(eng._h, int(base_step), int(alloc), int(resv), _timing._raw_stream(_timing._cur_dev()))
    if rc < 0:
        print(f"[TraceML] step memory not published (status {rc})", file=sys.stderr)


class trace_step:
    """``with trace_step(model): ...`` -- one training step."""

    __slots__ = ("model", "tracker", "region", "flags", "active", "t0", "mem_dev", "prev", "fast", "captured")

    def __init__(self, model):
        self.model = model
        self.active = not disabled()
        self.tracker = None
        self.region = None
        self.flags = None
        self.fast = None
        self.captured = False

    def __enter__(self):
        if not self.active:
            return self
        patches = _patches
        fast = _timing._FAST
        if fast is None and _timing._ENG is None:
            try:
                _timing._resolve()
                fast = _timing._FAST
            except _timing._Quiet:
                pass  # reported once by _resolve
            except Exception as exc:
                _log("engine start failed", exc)
        if _timing.GRAPH_SCOPE.depth and _timing._ENG is not None and self._enter_captured():
            return self
        if fast is not None:
            # fast path: same sequence as below with the three context managers and
            # the tracker object folded into this one (no per-step allocations)
            self.fast = fast
            try:
                info = _model_info(self.model)
                self.mem_dev = info[0]
                if info[0] >= 0:
                    fast.reset_peaks(info[0])
                t = patches._TLS
                self.prev = (t.fwd, t.fwd_depth, t.fwd_targets)
                t.fwd, t.fwd_depth, t.fwd_targets = True, 0, info[1]
                t.bwd = True
                t.h2d = True
                if _auto_optimizer():
                    patches.ensure_optimizer_timing_installed()
            except Exception as exc:
                _log("step setup failed", exc)
                self.prev = None
                self.mem_dev = -1
            self.t0 = _perf_ns()
            return self

        try:
            self.tracker = StepMemoryTracker(self.model)
            self.tracker.reset()
        except Exception as exc:
            _log("reset failed", exc)
        self.region = timed_region(STEP, "step", False)
        self.region.__enter__()
        self.flags = patches.step_auto_timers(self.model)
        self.flags.__enter__()
        try:
            if _auto_optimizer():
                patches.ensure_optimizer_timing_installed()
        except Exception as exc:
            _log("optimizer hook install failed", exc)
        return self

    def _enter_captured(self) -> bool:
        """A capturing stream inside trace_graph: open a captured step (False: not one)."""
        try:
            if not _capturing():
                return False
            eng = _timing._ENG
            slot = eng._gsbegin(eng._h, _timing._raw_stream(_timing._cur_dev()))
            if slot < 0:
                print(f"[TraceML] captured step not opened (status {slot})", file=sys.stderr)
                return False
            self.captured = True
            info = _model_info(self.model)
            self.mem_dev = info[0]
            t = _patches._TLS
            self.prev = (t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.bwd_depth, t.h2d)
            t.fwd, t.fwd_depth, t.fwd_targets = True, 0, info[1]
            t.bwd = True
            t.h2d = True
            if _auto_optimizer():
                _patches.ensure_optimizer_timing_installed()
        except Exception as exc:
            _log("captured step setup failed", exc)
        return self.captured

    def _exit_captured(self, exc_type) -> None:
        try:
            t = _patches._TLS
            if self.prev is not None:
                t.fwd, t.fwd_depth, t.fwd_targets, t.bwd, t.bwd_depth, t.h2d = self.prev
                self.prev = None
            eng = _timing._ENG
            flags = (FLAG_HAS_MEM if self.mem_dev >= 0 else 0) | (0 if exc_type is None else TML_GRAPH_STEP_FAILED)
            rc = eng._gscommit(eng._h, flags, _timing._raw_stream(_timing._cur_dev()))
            if rc < 0:
                print(f"[TraceML] captured step not committed (status {rc})", file=sys.stderr)
                return
            _timing.DEVICE_STEPS = True
            _timing.GRAPH_SCOPE.steps += 1
            _layers = sys.modules.get("traceml_b200.instrumentation.layers")
            if _layers is not None and _layers._PROFILES:
                _layers.commit_all_graph()
        except Exception as e:
            _log("captured step commit failed", e)
        finally:
            self.captured = False

    def __exit__(self, exc_type, exc, tb):
        if not self.active:
            return False
        if self.captured:
            self._exit_captured(exc_type)
            return False
        fast = self.fast
        if fast is not None:
            dur = _perf_ns() - self.t0
            try:
                t = _patches._TLS
                if self.prev is not None:
                    t.fwd, t.fwd_depth, t.fwd_targets = self.prev
                t.bwd, t.bwd_depth = False, 0
                t.h2d = False
                fast.host(PHASE_STEP, dur)
                if exc_type is None:
                    _STATE.advance_step()
                if _timing.DEVICE_STEPS:  # the device counts: send "advanced or not"
                    rc = fast.commit(int(exc_type is None), self.mem_dev, _wall())
                    if rc < 0:
                        _timing._ENG.step_discard()
                        print(f"[TraceML] step not committed (status {rc})", file=sys.stderr)
                    _publish(_timing._ENG, self.mem_dev)
                    _layers = sys.modules.get("traceml_b200.instrumentation.layers")
                    if _layers is not None and _layers._PROFILES:
                        _layers.commit_all(0)
                    return False
                rc = fast.commit(_STATE.step, self.mem_dev, _wall())
                if rc < 0:
                    _timing._ENG.step_discard()
                    print(f"[TraceML] step {_STATE.step} not committed (status {rc})", file=sys.stderr)
                _layers = sys.modules.get("traceml_b200.instrumentation.layers")
                if _layers is not None and _layers._PROFILES:  # deep profile: per-layer step close
                    _layers.commit_all(_STATE.step)
            except Exception as e:
                _log("flush failed", e)
            return False
        self.flags.__exit__(exc_type, exc, tb)
        self.region.__exit__(exc_type, exc, tb)
        state = get_trace_session_state()
        if exc_type is None:
            state.advance_step()
        try:
            if self.tracker is not None:
                self.tracker.record()
        except Exception as e:
            _log("record failed", e)
        device_steps = _timing.DEVICE_STEPS
        try:  # device-committed mode: the commit's step id only says "advanced or not"
            flush_step_events(self.model, int(exc_type is None) if device_steps else state.step)
        except Exception as e:
            _log("flush failed", e)
        if device_steps:
            try:
                _publish(_timing._ENG, self.tracker.index if self.tracker is not None and self.tracker.is_cuda else -1)
            except Exception as e:
                _log("step memory publish failed", e)
        return False


class trace_graph:
    """``with trace_graph(model): ...`` around a CUDA-graph capture of training work::

        g = torch.cuda.CUDAGraph()
        with traceml.trace_graph(model), torch.cuda.graph(g):
            loss = model(static_x).loss; loss.backward(); opt.step()
        for batch in loader:
            with traceml.trace_step(model):
                static_x.copy_(batch); g.replay()

    Arms the forward / backward / h2d openers of ``trace_step`` for the capture, and lets every
    device-timed region opened on a capturing stream (those, the optimizer hooks, ``trace_time``
    regions, deep-profile layers) capture its stamps into the graph.  Each replay then adds those
    regions' durations and calls to the step open on the device when it runs.  Opens no step and
    commits nothing.  Do not wrap ``torch.cuda.make_graphed_callables`` in it: its replays already
    run through the module and backward openers, so their regions would count twice.

    A ``trace_step`` inside the capture is a captured step instead: every replay commits one step
    per captured ``trace_step`` (see the module docstring), so the loop is only ``g.replay()``::

        with traceml.trace_graph(model), torch.cuda.graph(g):
            for _ in range(k):
                with traceml.trace_step(model):
                    loss = model(static_x).loss; loss.backward(); opt.step()
        for batch in loader:
            static_x.copy_(batch); g.replay()        # k step records

    The step records' memory is the allocator's current bytes as published at this scope's exit
    and after every host step: allocations made between replays are in no captured step."""

    __slots__ = ("model", "flags", "steps0")

    def __init__(self, model=None):
        self.model = model
        self.flags = None
        self.steps0 = 0

    def __enter__(self):
        if disabled():
            return self
        if _timing._ENG is None:
            # the engine's first region allocates device memory: never inside the capture
            try:
                _timing._resolve()
            except _timing._Quiet:
                pass  # reported once by _resolve
            except Exception as exc:
                _log("engine start failed", exc)
        self.flags = _patches.step_auto_timers(self.model)
        self.flags.__enter__()
        _timing.GRAPH_SCOPE.depth += 1
        _timing.GRAPH_SCOPES_OPEN[0] += 1
        self.steps0 = _timing.GRAPH_SCOPE.steps
        try:
            if _auto_optimizer():
                _patches.ensure_optimizer_timing_installed()
        except Exception as exc:
            _log("optimizer hook install failed", exc)
        return self

    def __exit__(self, exc_type, exc, tb):
        if self.flags is None:
            return False
        _timing.GRAPH_SCOPES_OPEN[0] -= 1
        _timing.GRAPH_SCOPE.depth -= 1
        self.flags.__exit__(exc_type, exc, tb)
        self.flags = None
        if _timing.GRAPH_SCOPE.steps != self.steps0 and _timing._ENG is not None:
            # steps were captured: memory for their replays, and the id they continue from
            try:
                eng = _timing._ENG
                base = _STATE.step
                _publish(eng, _model_info(self.model)[0] if self.model is not None else eng.device, base)
                _STATE.bind_device_step(eng.graph_step_id)
            except Exception as e:
                _log("captured steps setup failed", e)
        return False


def trace_model_instance(model, sample_layer_memory: bool = True, trace_layer_forward_memory: bool = True,
                         trace_layer_backward_memory: bool = True, trace_layer_forward_time: bool = True,
                         trace_layer_backward_time: bool = True, trace_execution: bool = True,
                         include_names=None, exclude_names=None, leaf_only: bool = True) -> None:
    """Deep (per-layer) profile: forward / backward device timers and activation sizes per leaf
    module, same signature and gate as ``sdk/instrumentation.py:203-260`` (``TRACEML_PROFILE=deep``;
    a no-op otherwise).  K1 / K2 with a layer id: ``instrumentation/layers.py``."""
    if disabled() or (os.environ.get("TRACEML_PROFILE", "run") or "run").strip().lower() != "deep":
        return
    try:
        import torch.nn as nn

        if not isinstance(model, nn.Module):
            raise TypeError("trace_model_instance expects an nn.Module.")
        from ..instrumentation import layers
        from ..runtime import get_engine

        layers.attach(get_engine(), model, include_names=include_names, exclude_names=exclude_names,
                      leaf_only=leaf_only,
                      forward=bool(trace_layer_forward_time or trace_layer_forward_memory),
                      backward=bool(trace_layer_backward_time or trace_layer_backward_memory))
    except Exception as exc:  # noqa: BLE001 -- never into user code
        _log("trace_model_instance failed", exc)


def trace_time(name: str, scope: str = "global", use_gpu: bool = True) -> Callable:
    if disabled():
        return lambda func: func
    if scope not in ("step", "global"):
        raise ValueError(f"Invalid scope {scope!r}. Expected 'step' or 'global'.")

    def decorator(func: Callable):
        @functools.wraps(func)
        def wrapper(*args, **kwargs):
            with timed_region(name, scope=scope, use_gpu=use_gpu):
                return func(*args, **kwargs)

        return wrapper

    return decorator


class _TraceStateMeta(type):
    @property
    def step(cls) -> int:
        return get_trace_session_state().step

    @step.setter
    def step(cls, value: int) -> None:
        get_trace_session_state().set_step(value)


class TraceState(metaclass=_TraceStateMeta):
    """Compatibility facade (``TraceState.step += 1`` keeps working)."""

    @classmethod
    def reset(cls, step: int = 0) -> int:
        return get_trace_session_state().reset(step)

    @classmethod
    def advance(cls, delta: int = 1) -> int:
        return get_trace_session_state().advance_step(delta)


__all__ = ["trace_step", "trace_graph", "trace_model_instance", "trace_time", "TraceState"]
