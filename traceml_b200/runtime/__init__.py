"""Per-rank runtime: the engine singleton and the sampler agent.

Replaces ``src/traceml/runtime/runtime.py:33-193`` (TraceMLRuntime) and the
sampler registry's ``run`` profile (``runtime/sampler_registry.py:78-160``):
one native engine per process/GPU instead of three Python samplers fed by
queues.  The sampler thread here only drains the host-mapped mirror (no CUDA
call) and takes the 1 kHz process samples; it never touches the training
stream.
"""
from __future__ import annotations

import os
import sys
import threading
import time
from typing import Any, Callable, Dict, List, Optional

from .state import TraceSessionState, get_trace_session_state, reset_trace_session_state

_LOCK = threading.Lock()
_ENGINE = None
_ENGINE_DEVICE: Optional[int] = None


_DISABLED = os.environ.get("TRACEML_DISABLED", "0") == "1"


def disabled() -> bool:
    """TRACEML_DISABLED=1 short-circuits every hook.  Read once at import, like the
    reference's module constants (utils/timing.py:28): the per-region check must not
    cost an ``os.environ`` lookup."""
    return _DISABLED


def refresh_disabled() -> bool:
    global _DISABLED
    _DISABLED = os.environ.get("TRACEML_DISABLED", "0") == "1"
    return _DISABLED


def summary_window_rows() -> int:
    try:
        return max(1, int(os.environ.get("TRACEML_SUMMARY_WINDOW_ROWS", "10000")))
    except ValueError:
        return 10_000


def _identity():
    """Global rank / world size without touching CUDA (runtime/identity.py:135-234)."""
    rank = int(os.environ.get("RANK", "0") or 0)
    world = int(os.environ.get("WORLD_SIZE", "1") or 1)
    try:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            rank, world = dist.get_rank(), dist.get_world_size()
    except Exception:
        pass
    return rank, world


def get_engine(device: Optional[int] = None):
    """The process's engine, created on first use on the current CUDA device.

    Raises if there is no CUDA device or the native library is missing: the
    GPU engine has no CPU fallback.
    """
    global _ENGINE, _ENGINE_DEVICE
    if _ENGINE is not None and (device is None or device == _ENGINE_DEVICE):
        return _ENGINE
    with _LOCK:
        if _ENGINE is not None and (device is None or device == _ENGINE_DEVICE):
            return _ENGINE
        import torch

        if not torch.cuda.is_available():
            raise RuntimeError(
                "traceml_b200: no CUDA device is visible. The GPU-native telemetry engine "
                "records through CUDA kernels and has no CPU fallback.")
        from ..engine import Engine

        dev = torch.cuda.current_device() if device is None else int(device)
        rank, world = _identity()
        window = summary_window_rows()
        # reference retention: 1.5 x window rows per rank (reporting/config.py:13-35)
        slots = int(os.environ.get("TRACEML_RING_SLOTS", str(int(window * 1.5))))
        if _ENGINE is not None:
            import sys as _sys

            timing = _sys.modules.get("traceml_b200.utils.timing")
            if timing is not None:
                timing._reset()  # unbind the fast path + join the sampler before the context goes
            _ENGINE.close()
        _ENGINE = Engine(device=dev, rank=rank, world=world, ring_slots=max(1, slots),
                         proc_slots=max(1, slots))
        _ENGINE_DEVICE = dev
        return _ENGINE


def peek_engine():
    """The process engine if the training thread has created it, else None.  Side threads
    (sampler, render tick) use this: only the training thread -- whose current CUDA device is
    the rank's device -- may create the engine."""
    return _ENGINE


def shutdown_engine() -> None:
    """Join the native sampler, unbind the step glue, then free the context -- in that order:
    the sampler thread and the bound fast path hold raw pointers into the context."""
    global _ENGINE, _ENGINE_DEVICE
    with _LOCK:
        import sys

        timing = sys.modules.get("traceml_b200.utils.timing")
        if timing is not None:
            timing._reset()
        if _ENGINE is not None:
            _ENGINE.close()
        _ENGINE = None
        _ENGINE_DEVICE = None


import atexit as _atexit

# a run that raises, or never calls TraceMLRuntime.stop(), must still join the native sampler
# before static destruction (a joinable std::thread at exit is std::terminate)
_atexit.register(shutdown_engine)


class TraceMLRuntime:
    """Sampler agent: every ``interval`` seconds take one process sample and
    hand newly completed step records to the registered sinks.

    ``sinks`` are callables ``sink(kind, rows)`` with ``kind`` in
    {"step_time", "step_memory", "process"} and ``rows`` the reference's wire
    rows (samplers/schema/*.py) -- this is where the kept TCP publisher /
    aggregator attaches (INTEGRATION.md).
    """

    def __init__(self, interval_sec: float = 2.0, sinks: Optional[List[Callable]] = None,
                 sample_process: bool = True, native_process_hz: float = 0.0,
                 sample_system: Optional[bool] = None):
        self.interval = max(1e-4, float(interval_sec))
        self.sinks = list(sinks or [])
        self.sample_process = sample_process
        # > 0: the C++ sampler thread (no GIL) commits process samples at this rate and the
        # Python tick only drains; 0: one sample per tick from Python (the reference cadence)
        self.native_process_hz = float(native_process_hz)
        # host / NVML snapshot: local rank 0 only, like the reference's registry
        # (runtime/sampler_registry.py:78-105); None = decide from LOCAL_RANK
        self.sample_system = (int(os.environ.get("LOCAL_RANK", "0") or 0) == 0) if sample_system is None \
            else bool(sample_system)
        self._sys = None
        self._sys_stream = None
        self._native = None
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._proc = None
        self.ticks = 0
        self.steps_seen = 0
        self.dropped = 0

    def start(self) -> None:
        if disabled() or self._thread is not None:
            return
        from ..samplers import ProcessProbe

        self._proc = None
        if self.sample_system and self._sys is None:
            # NVML / psutil set-up here, not inside a tick: initialising NVML holds the driver for
            # long enough to stall the native sampler's launches and the training thread's
            try:
                from ..samplers import SystemProbe

                self._sys = SystemProbe()
            except Exception as exc:  # noqa: BLE001 -- samplers never interfere with training
                print(f"[TraceML] system probe unavailable: {exc}", file=sys.stderr)
        if self.sample_process and self.native_process_hz > 0:
            from ..utils import timing

            timing._ENG or timing._resolve()
            if timing._FAST is None:
                raise RuntimeError("native process sampler needs the _tml_step extension")
            self._native = timing._FAST
            self._native.sampler_start(int(round(1.0e6 / self.native_process_hz)), 0)
        elif self.sample_process:
            self._proc = ProcessProbe()
        self._thread = threading.Thread(target=self._loop, name="traceml-b200-sampler", daemon=True)
        self._thread.start()

    def _tick(self) -> None:
        from ..samplers import drain_to_wire

        # never create the engine here: a new host thread's current device is 0, so an engine
        # created from the sampler thread would land on cuda:0 for every rank
        eng = peek_engine()
        if eng is None:
            return
        if self._proc is not None:
            if not self._proc._cuda_safe():
                return  # distributed job before init_process_group (process_sampler.py:150-158)
            import torch

            with torch.cuda.device(eng.device):
                self._proc.sample(eng)
        out = drain_to_wire(eng, ram_total=getattr(self._proc, "ram_total", None))
        out["system"] = []
        if self.sample_system:
            # with or without sinks (the reference's registry samples regardless): the snapshot goes
            # into the engine's system ring for the final summary, and its wire row to the sinks
            try:
                if self._sys is None:
                    from ..samplers import SystemProbe

                    self._sys = SystemProbe()  # start() could not make one: try again
                row, rec = self._sys.snapshot()
                out["system"] = [row]
                import torch

                if self._sys_stream is None:
                    self._sys_stream = torch.cuda.Stream(device=eng.device)  # never the training stream
                eng.sys_commit(rec, int(self._sys_stream.cuda_stream))
            except Exception as exc:  # noqa: BLE001
                print(f"[TraceML] system sample failed: {exc}", file=sys.stderr)
        self.steps_seen += len(out["step_time"])
        self.dropped += out["dropped"]
        self.ticks += 1
        for sink in self.sinks:
            for kind in ("step_time", "step_memory", "process", "system"):
                if out[kind]:
                    try:
                        sink(kind, out[kind])
                    except Exception as exc:  # fail-open (runtime/sender.py:132-139)
                        print(f"[TraceML] sink failed: {exc}", file=sys.stderr)

    def _loop(self) -> None:
        while not self._stop.wait(self.interval):
            try:
                self._tick()
            except Exception as exc:
                print(f"[TraceML] sampler tick failed: {exc}", file=sys.stderr)

    def stop(self) -> None:
        if self._thread is None:
            return
        self._stop.set()
        self._thread.join(timeout=5.0)
        self._thread = None
        if self._native is not None:
            self.native_samples, self.native_late = self._native.sampler_stop()
            self._native = None
        try:
            self._tick()  # final drain (runtime/runtime.py:163-193)
        except Exception as exc:
            print(f"[TraceML] final tick failed: {exc}", file=sys.stderr)


__all__ = ["TraceMLRuntime", "TraceSessionState", "get_engine", "peek_engine", "shutdown_engine", "disabled", "refresh_disabled",
           "get_trace_session_state", "reset_trace_session_state", "summary_window_rows"]
