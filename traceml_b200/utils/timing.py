"""Phase timer seam (mirror of ``src/traceml/utils/timing.py:44-256``).

Same names and call semantics as the reference -- ``timed_region(name, scope,
use_gpu)``, ``TimeEvent``, ``TimeScope``, ``record_event``,
``flush_step_time_buffer`` -- but a region is two 1-warp ``%globaltimer`` stamp
kernels on the current stream (``tml_phase_begin`` / ``tml_phase_end``) that
accumulate into the open step's in-flight record on the device.  There are no
CUDA events, no event pool, no Python event objects and no queue; nothing here
synchronises the host with the GPU.

Semantics kept (SURVEY 8a): repeated regions within a step sum and count
``n_calls``; ``use_gpu=False`` regions are host-clock; GLOBAL-scope regions run
but are not recorded (``utils/timing.py:123-134`` drops them too); telemetry
errors never reach user code.

Under CUDA-graph capture the stamp entry points return ``TML_ERR_CAPTURE`` and the
region takes the host clock, unless a ``trace_graph`` scope is open on this thread:
then the stamps are captured into the graph (``tml_graph_phase_begin`` / ``_end``)
and time the region on every replay.

Once a step commit has been captured (``DEVICE_STEPS``), replays commit steps on the
device, and host-clock regions are added there too (``tml_graph_phase_host``): to
the step the device has open when they run, so input waits between replays land in
the step the next replay commits.
"""
from __future__ import annotations

import os
import sys
import threading
import time
from dataclasses import dataclass
from enum import Enum
from typing import Any, Optional

from .._abi import TML_ERR_CAPTURE
from ..records import (PHASE_BACKWARD, PHASE_DATALOADER, PHASE_EVENT_NAMES, PHASE_FORWARD,
                       PHASE_OPTIMIZER, PHASE_STEP)
from ..runtime import disabled, get_engine

PHASE_OTHER = 6
_PHASE_BY_NAME = {n: i for i, n in enumerate(PHASE_EVENT_NAMES)}
_perf_ns = time.perf_counter_ns
_raw_stream = None  # torch._C._cuda_getCurrentRawStream, bound lazily
_cur_dev = None
_ENG = None         # the process engine, resolved on first use
_FAST = None        # traceml_b200._tml_step bound to that engine (None: ctypes path)


_RESOLVE_FAILED: Optional[str] = None  # a failed engine resolution is cached and printed once

# A region captured into a CUDA graph (tml_graph_phase_begin) keeps its graph slot g in ``slot`` as
# GRAPH_SLOT0 - g: below every status code, so the plain path's ``slot >= 0`` test is unchanged.
GRAPH_SLOT0 = -(1 << 16)


class _GraphScope(threading.local):
    depth = 0   # open trace_graph scopes on this thread
    steps = 0   # step commits this thread captured (trace_graph publishes memory when it grew)


GRAPH_SCOPE = _GraphScope()
GRAPH_SCOPES_OPEN = [0]  # open trace_graph scopes in the process (layer backward hooks run on
                         # autograd's device thread, not on the thread that opened the scope)
DEVICE_STEPS = False     # the engine is in device-committed mode (a step commit was captured)


def _resolve():
    """First region of the process: create the engine, bind the native step glue."""
    global _ENG, _FAST, _RESOLVE_FAILED
    if _RESOLVE_FAILED is not None:
        raise _Quiet(_RESOLVE_FAILED)
    try:
        eng = get_engine()
    except Exception as exc:
        _RESOLVE_FAILED = f"{type(exc).__name__}: {exc}"
        print(f"[TraceML] telemetry engine unavailable, regions are not recorded: {_RESOLVE_FAILED}",
              file=sys.stderr)
        raise _Quiet(_RESOLVE_FAILED) from exc
    if _raw_stream is None:
        _bind_torch()
    fast = None
    try:
        from .. import _abi, _tml_step

        _tml_step.bind(_abi.LIB_PATH, int(eng._h.value), int(eng.device))
        fast = _tml_step
    except Exception as exc:
        print(f"[TraceML] native step glue unavailable ({exc}); using the ctypes path", file=sys.stderr)
    _ENG, _FAST = eng, fast
    return eng


class _Quiet(RuntimeError):
    """Engine resolution already failed and was reported: callers stay silent."""


def _reset() -> None:
    global _ENG, _FAST, _RESOLVE_FAILED, DEVICE_STEPS
    _RESOLVE_FAILED = None
    if DEVICE_STEPS:
        from ..runtime import get_trace_session_state

        get_trace_session_state().bind_device_step(None)
        DEVICE_STEPS = False
    if _FAST is not None:
        try:
            _FAST.unbind()
        except Exception:
            pass
    _ENG, _FAST = None, None


class TimeScope(str, Enum):
    STEP = "step"
    GLOBAL = "global"


@dataclass
class TimeEvent:
    """Compatibility carrier for hand-made events (integrations/lightning.py:160-174)."""

    name: str
    device: str = "cpu"
    cpu_start: float = 0.0
    cpu_end: float = 0.0
    gpu_start: Any = None
    gpu_end: Any = None
    gpu_time_ms: Optional[float] = None
    resolved: bool = False
    step: int = -1
    scope: TimeScope = TimeScope.STEP


def phase_of(name: str) -> int:
    """Event name -> phase id.  Canonical names map directly; other names use the
    reference's bucket rules (reporting/sections/step_time/model.py:50-74);
    anything else is timed into the unsummarised OTHER slot."""
    p = _PHASE_BY_NAME.get(name)
    if p is not None:
        return p
    n = str(name).lower()
    if "step_time" in n:
        return PHASE_STEP
    if "dataloader_next" in n:
        return PHASE_DATALOADER
    if "forward_time" in n:
        return PHASE_FORWARD
    if "backward_time" in n:
        return PHASE_BACKWARD
    if "optimizer_step" in n:
        return PHASE_OPTIMIZER
    if "h2d_time" in n:
        return 1
    if "data" in n or "input" in n or "batch" in n:
        return PHASE_DATALOADER
    if "forward" in n or n == "fwd":
        return PHASE_FORWARD
    if "backward" in n or "bwd" in n:
        return PHASE_BACKWARD
    if "optim" in n or n in {"step", "update"}:
        return PHASE_OPTIMIZER
    return PHASE_OTHER


def _bind_torch():
    global _raw_stream, _cur_dev
    import torch

    _raw_stream = torch._C._cuda_getCurrentRawStream
    _cur_dev = torch.cuda.current_device


class timed_region:
    """Context manager timing one region.  Class-based (not a generator) so the
    per-region host cost is two C calls plus a handful of attribute writes."""

    __slots__ = ("phase", "gpu", "record", "slot", "t0", "eng", "on")

    def __init__(self, name: str, scope: Any = TimeScope.STEP, use_gpu: bool = True):
        self.phase = phase_of(name)
        self.gpu = bool(use_gpu)
        sc = scope.value if isinstance(scope, TimeScope) else str(scope)
        self.on = (sc == "step") and not disabled()  # static: does this region record at all
        self.record = self.on                        # per use: cleared when one setup fails
        self.slot = -1
        self.t0 = 0
        self.eng = None

    def __enter__(self):
        # region objects are reused (instrumentation/patches.py): one failed setup must not
        # silence the phase for the rest of the process
        self.record = self.on
        self.slot = -1
        if not self.record:
            return self
        try:
            eng = self.eng = _ENG or _resolve()
            if self.gpu:
                fast = _FAST
                if fast is not None:
                    self.slot = fast.begin(self.phase)
                else:
                    self.slot = eng._begin(eng._h, self.phase, _raw_stream(_cur_dev()))
                if self.slot < 0:
                    if self.slot == TML_ERR_CAPTURE and GRAPH_SCOPE.depth:  # inside trace_graph
                        g = eng._gbegin(eng._h, self.phase, _raw_stream(_cur_dev()))
                        if g >= 0:
                            self.slot = GRAPH_SLOT0 - g
                            return self
                    self.t0 = _perf_ns()  # graph capture / launch failure: host clock
            else:
                self.t0 = _perf_ns()
        except _Quiet:
            self.record = False
        except Exception as exc:  # timing setup failed: user code still runs
            self.record = False
            print(f"[TraceML] timed_region setup failed: {exc}", file=sys.stderr)
        return self

    def __exit__(self, exc_type, exc, tb):
        if not self.record:
            return False
        try:
            fast = _FAST
            if fast is not None:
                if self.slot >= 0:
                    fast.end(self.phase, self.slot)
                elif self.slot > GRAPH_SLOT0:
                    if DEVICE_STEPS:
                        _device_host(self.eng, self.phase, _perf_ns() - self.t0)
                    else:
                        fast.host(self.phase, _perf_ns() - self.t0)
                else:
                    self._graph_end()
            else:
                eng = self.eng
                if self.slot >= 0:
                    eng._end(eng._h, self.phase, self.slot, _raw_stream(_cur_dev()))
                elif self.slot > GRAPH_SLOT0:
                    if DEVICE_STEPS:
                        _device_host(eng, self.phase, _perf_ns() - self.t0)
                    else:
                        eng._host(eng._h, self.phase, _perf_ns() - self.t0)
                else:
                    self._graph_end()
        except Exception as e:  # nothing here may break training
            print(f"[TraceML] timed_region teardown failed: {e}", file=sys.stderr)
        return False

    def _graph_end(self):
        eng = self.eng
        rc = eng._gend(eng._h, self.phase, GRAPH_SLOT0 - self.slot, _raw_stream(_cur_dev()))
        if rc < 0:
            print(f"[TraceML] graph region not closed (status {rc})", file=sys.stderr)


def _device_host(eng, phase: int, dur_ns: int) -> None:
    """A host-clock duration in device-committed mode: added on the device, in stream order."""
    eng._ghost(eng._h, phase, max(0, int(dur_ns)), _raw_stream(_cur_dev()))


def record_event(evt: TimeEvent) -> None:
    """Record an already-measured event (host duration) into the open step."""
    if disabled():
        return
    scope = evt.scope.value if isinstance(evt.scope, TimeScope) else str(evt.scope)
    if scope != "step":
        return
    try:
        ms = evt.gpu_time_ms if evt.gpu_time_ms is not None else (evt.cpu_end - evt.cpu_start) * 1000.0
        eng = _ENG or _resolve()
        dur = max(0, int(round(float(ms) * 1.0e6)))
        if DEVICE_STEPS:
            _device_host(eng, phase_of(evt.name), dur)
        else:
            eng._host(eng._h, phase_of(evt.name), dur)
    except _Quiet:
        pass
    except Exception as exc:
        print(f"[TraceML] record_event failed: {exc}", file=sys.stderr)


def flush_step_time_buffer(step: int) -> None:
    """Kept for seam compatibility (utils/timing.py:163-180).  The in-flight
    record is committed by ``flush_step_events`` together with the memory
    peaks -- one commit kernel per step -- so there is nothing to move here."""
    return None


__all__ = ["TimeScope", "TimeEvent", "timed_region", "record_event", "flush_step_time_buffer",
           "phase_of", "PHASE_OTHER"]
