"""traceml_b200 -- GPU-native (H100) per-step telemetry + cross-rank diagnostics engine.

Drop-in for the hot path of traceopt-ai/traceml (v0.2.15): the per-step phase
timers, the step/process memory samplers and the cross-rank step-alignment /
rank-skew reduce behind the Step-Time, Step-Memory and Process diagnoses.

The public surface mirrors ``src/traceml/api.py:11-135`` of the reference::

    import traceml_b200 as traceml
    traceml.init(mode="auto")
    for batch in loader:
        with traceml.trace_step(model):
            ...

Submodules that only describe data (``records``) import without
the CUDA extension; everything that records or reduces telemetry loads
``libtraceml_b200.so`` and raises if it is missing -- there is no CPU fallback.
"""

from __future__ import annotations

__version__ = "0.1.0"

_LAZY = {
    "init": ("traceml_b200.sdk", "init"),
    "start": ("traceml_b200.sdk", "start"),
    "trace_step": ("traceml_b200.sdk", "trace_step"),
    "trace_graph": ("traceml_b200.sdk", "trace_graph"),
    "trace_time": ("traceml_b200.sdk", "trace_time"),
    "trace_model_instance": ("traceml_b200.sdk", "trace_model_instance"),
    "wrap_dataloader_fetch": ("traceml_b200.sdk", "wrap_dataloader_fetch"),
    "wrap_forward": ("traceml_b200.sdk", "wrap_forward"),
    "wrap_backward": ("traceml_b200.sdk", "wrap_backward"),
    "wrap_optimizer": ("traceml_b200.sdk", "wrap_optimizer"),
    "wrap_h2d": ("traceml_b200.sdk", "wrap_h2d"),
    "final_summary": ("traceml_b200.summary", "final_summary"),
    "TraceMLInitConfig": ("traceml_b200.sdk", "TraceMLInitConfig"),
}


def __getattr__(name: str):
    target = _LAZY.get(name)
    if target is None:
        raise AttributeError(f"module 'traceml_b200' has no attribute {name!r}")
    import importlib

    return getattr(importlib.import_module(target[0]), target[1])


__all__ = sorted(_LAZY) + ["__version__"]
