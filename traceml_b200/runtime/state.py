"""Process-local step counter (mirror of ``src/traceml/runtime/state.py:17-98``).

The semantic step is TraceML's own counter: it advances once per completed
``trace_step`` (so gradient-accumulation micro-batches count), the first
recorded step id is 1, and reports use ``training_steps = max(step) + 1``.
"""
from __future__ import annotations

from threading import RLock


class TraceSessionState:
    __slots__ = ("_step", "_lock", "_device_step")

    def __init__(self, initial_step: int = 0) -> None:
        self._lock = RLock()
        self._step = self._check(initial_step)
        self._device_step = None

    @staticmethod
    def _check(value: int) -> int:
        if not isinstance(value, int) or isinstance(value, bool):
            raise TypeError("TraceML step must be an integer.")
        if value < 0:
            raise ValueError("TraceML step must be non-negative.")
        return value

    @property
    def step(self) -> int:
        """The last step id.  Once a step commit has been captured into a CUDA graph the replays
        create the steps on the device, and this reads the device's last id (one 8-B copy)."""
        read = self._device_step
        if read is not None:
            return read()
        with self._lock:
            return self._step

    def bind_device_step(self, read) -> None:
        """``read()`` returns the device's last step id from now on (None: the host counter again)."""
        self._device_step = read

    def set_step(self, value: int) -> int:
        v = self._check(value)
        with self._lock:
            self._step = v
            return v

    def advance_step(self, delta: int = 1) -> int:
        if not isinstance(delta, int) or isinstance(delta, bool):
            raise TypeError("TraceML step delta must be an integer.")
        if delta < 0:
            raise ValueError("TraceML step delta must be non-negative.")
        with self._lock:
            self._step = self._check(self._step + delta)
            return self._step

    def reset(self, step: int = 0) -> int:
        return self.set_step(step)


_STATE = TraceSessionState()


def get_trace_session_state() -> TraceSessionState:
    return _STATE


def reset_trace_session_state(step: int = 0) -> int:
    return _STATE.reset(step)


__all__ = ["TraceSessionState", "get_trace_session_state", "reset_trace_session_state"]
