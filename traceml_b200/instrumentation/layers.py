"""Deep profile: per-layer forward / backward device timers and activation sizes (SURVEY 8f-4).

Replaces ``instrumentation/hooks/layer_forward_time_hooks.py:113-267``,
``layer_backward_time_hooks.py:110-264`` (two pooled CUDA events + one event object per layer call,
resolved later by ``event.query()``) and the output-size bookkeeping of
``layer_forward_memory_hooks.py:60-190`` / ``layer_backward_memory_hooks.py`` with K1 / K2 carrying
a layer id: a layer call is two 1-warp ``%globaltimer`` stamps on the current stream
(``tml_layer_begin`` / ``tml_layer_end``) that accumulate duration, call count and the call's
output bytes into the layer's device accumulators; ``tml_layer_commit`` at the step boundary
snapshots all layers into a device ring, ``tml_layer_drain`` (sampler side, own stream) brings
finished steps to the host.  No events, no queues, no host synchronisation on the training thread.
While a ``trace_graph`` scope is open, a layer call on a capturing stream captures its stamps into
the graph (``tml_graph_layer_begin`` / ``_end``), so every replay adds to the layer's records; the
scope is checked process-wide because backward hooks run on autograd's device thread.

Which modules are hooked is the reference's decision logic (``utils/shared_utils.py:11-37``): leaf
modules by default, ``include_names`` / ``exclude_names`` substring filters.  Hooks are attached
only under ``TRACEML_PROFILE=deep`` (``sdk/instrumentation.py:222``).
"""
from __future__ import annotations

import ctypes as C
import sys
import time
from typing import Any, Dict, Iterable, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from .. import _abi
from ..utils.timing import GRAPH_SCOPES_OPEN, GRAPH_SLOT0

LAYER_RECORD_DTYPE = np.dtype([("step", "<u8"), ("fwd_ns", "<u8"), ("bwd_ns", "<u8"), ("fwd_calls", "<u4"),
                               ("bwd_calls", "<u4"), ("fwd_bytes", "<u8"), ("bwd_bytes", "<u8")])
assert LAYER_RECORD_DTYPE.itemsize == C.sizeof(_abi.LayerRecord) == 48


def get_hookable_modules(model: nn.Module, include_names: Optional[List[str]] = None,
                         exclude_names: Optional[List[str]] = None, leaf_only: bool = True
                         ) -> Iterable[Tuple[str, nn.Module]]:
    """utils/shared_utils.py:11-37, same filters in the same order."""
    for name, module in model.named_modules():
        if leaf_only and any(module.children()):
            continue
        if not leaf_only and name == "":
            continue
        if include_names and not any(inc in name for inc in include_names):
            continue
        if exclude_names and any(exc in name for exc in exclude_names):
            continue
        yield name, module


def _tensor_bytes(obj: Any) -> int:
    """Bytes of the tensors in a hook's output (layer_forward_memory_hooks.py:60-100: tensors,
    lists / tuples / dicts of tensors)."""
    if isinstance(obj, torch.Tensor):
        return obj.numel() * obj.element_size()
    if isinstance(obj, (list, tuple)):
        return sum(_tensor_bytes(o) for o in obj)
    if isinstance(obj, dict):
        return sum(_tensor_bytes(o) for o in obj.values())
    return 0


class LayerProfile:
    """Hooks + drain for one model on one engine."""

    def __init__(self, engine, model: nn.Module, include_names=None, exclude_names=None, leaf_only: bool = True,
                 ring_steps: int = 256, forward: bool = True, backward: bool = True, outermost: bool = False):
        """``outermost``: open the region before any hook registered earlier on the same module
        (pre-hooks are prepended); the closing hooks are appended, so with hooks attached LAST
        this profile brackets every other hook's work."""
        self.engine = engine
        self.model_id = id(model)
        self.names: List[str] = []
        self.handles: List[Any] = []
        self._lib = _abi.lib()
        mods = list(get_hookable_modules(model, include_names, exclude_names, leaf_only))
        self.names = [n for n, _ in mods]
        if not mods:
            return
        _abi.check(self._lib.tml_layer_init(engine._h, len(mods), int(ring_steps)), "tml_layer_init")
        raw_stream = torch._C._cuda_getCurrentRawStream
        dev = engine.device
        h, begin, end = engine._h, self._lib.tml_layer_begin, self._lib.tml_layer_end
        gbegin, gend = self._lib.tml_graph_layer_begin, self._lib.tml_graph_layer_end

        def graph_begin(status, stream):
            """A capturing stream inside trace_graph: the layer's stamps go into the graph."""
            if status == _abi.TML_ERR_CAPTURE and GRAPH_SCOPES_OPEN[0]:
                g = gbegin(h, stream)
                if g >= 0:
                    return GRAPH_SLOT0 - g
            return status

        for lid, (_, m) in enumerate(mods):
            slots: List[int] = []   # a module may be re-entered (shared layers): FIFO like the reference's deque
            bslots: List[int] = []

            def pre(mod, args, _s=slots):
                stream = raw_stream(dev)
                slot = begin(h, stream)
                _s.append(slot if slot >= 0 else graph_begin(slot, stream))

            def post(mod, args, out, _s=slots, _lid=lid):
                if _s:
                    slot = _s.pop(0)
                    if slot >= 0:
                        end(h, _lid, 0, slot, _tensor_bytes(out), raw_stream(dev))
                    elif slot <= GRAPH_SLOT0:
                        gend(h, _lid, 0, GRAPH_SLOT0 - slot, _tensor_bytes(out), raw_stream(dev))

            def bpre(mod, gout, _s=bslots):
                stream = raw_stream(dev)
                slot = begin(h, stream)
                _s.append(slot if slot >= 0 else graph_begin(slot, stream))

            def bpost(mod, gin, gout, _s=bslots, _lid=lid):
                if _s:
                    slot = _s.pop(0)
                    if slot >= 0:
                        end(h, _lid, 1, slot, _tensor_bytes(gout), raw_stream(dev))
                    elif slot <= GRAPH_SLOT0:
                        gend(h, _lid, 1, GRAPH_SLOT0 - slot, _tensor_bytes(gout), raw_stream(dev))

            if forward:
                self.handles.append(m.register_forward_pre_hook(pre, prepend=outermost))
                self.handles.append(m.register_forward_hook(post))
            if backward:
                self.handles.append(m.register_full_backward_pre_hook(bpre, prepend=outermost))
                self.handles.append(m.register_full_backward_hook(bpost))
        self._buf = np.zeros((8, len(mods)), dtype=LAYER_RECORD_DTYPE)
        self.seq = 0

    def commit(self, step: int) -> None:
        """Step boundary (flush_layer_*_buffers of utils/flush_buffers.py:24-33)."""
        if self.names:
            self._lib.tml_layer_commit(self.engine._h, int(step),
                                       torch._C._cuda_getCurrentRawStream(self.engine.device))

    def commit_graph(self) -> None:
        """The step boundary of a step captured into a CUDA graph: every replay closes the layers'
        step under the step id the device assigned."""
        if self.names:
            rc = self._lib.tml_graph_layer_commit(self.engine._h,
                                                  torch._C._cuda_getCurrentRawStream(self.engine.device))
            if rc < 0:
                print(f"[TraceML] layer step close not captured (status {rc})", file=sys.stderr)

    def drain(self) -> np.ndarray:
        """Finished steps as a ``[steps, layers]`` record array (sampler thread)."""
        if not self.names:
            return np.zeros((0, 0), dtype=LAYER_RECORD_DTYPE)
        n, nl, dropped = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        out = []
        while True:
            _abi.check(self._lib.tml_layer_drain(self.engine._h, self._buf.ctypes.data, self._buf.shape[0],
                                                 C.byref(n), C.byref(nl), C.byref(dropped)), "tml_layer_drain")
            if n.value:
                out.append(self._buf[: n.value].copy())
            if n.value < self._buf.shape[0]:
                break
        return np.concatenate(out) if out else np.zeros((0, len(self.names)), dtype=LAYER_RECORD_DTYPE)

    def wire_rows(self, recs: np.ndarray, device: Optional[str] = None) -> Dict[str, List[Dict[str, Any]]]:
        """The rows of the four reference layer tables (samplers/schema/
        layer_forward_backward_time.py:120-140, layer_forward_backward_memory.py): parallel lists,
        layers that were not called in a step are left out, like the reference's aggregation."""
        dev = device or f"cuda:{self.engine.device}"
        out: Dict[str, List[Dict[str, Any]]] = {"layer_forward_time": [], "layer_backward_time": [],
                                               "layer_forward_memory": [], "layer_backward_memory": []}
        now = time.time()
        for row in recs:
            self.seq += 1
            step = int(row["step"][0]) if len(row) else 0
            for tag, ns, calls, nbytes in (("forward", "fwd_ns", "fwd_calls", "fwd_bytes"),
                                           ("backward", "bwd_ns", "bwd_calls", "bwd_bytes")):
                idx = [i for i in range(len(self.names)) if int(row[calls][i]) > 0]
                if not idx:
                    continue
                base = {"seq": self.seq, "ts": now, "model_id": self.model_id, "step": step, "device": dev,
                        "layers": [self.names[i] for i in idx]}
                ms = [float(int(row[ns][i])) / 1.0e6 for i in idx]
                out[f"layer_{tag}_time"].append(dict(base, cpu_ms=ms, gpu_ms=list(ms),
                                                     n_calls=[int(row[calls][i]) for i in idx]))
                out[f"layer_{tag}_memory"].append(dict(base, memory=[float(int(row[nbytes][i])) for i in idx]))
        return out

    def detach(self) -> None:
        for h in self.handles:
            h.remove()
        self.handles = []


_PROFILES: Dict[int, LayerProfile] = {}


def attach(engine, model: nn.Module, **kw) -> LayerProfile:
    """One profile per model instance (the reference's hook registries: ``_layer_*_hook_registry``)."""
    p = _PROFILES.get(id(model))
    if p is None:
        p = _PROFILES[id(model)] = LayerProfile(engine, model, **kw)
    return p


def profile_of(model) -> Optional[LayerProfile]:
    return _PROFILES.get(id(model))


def commit_all(step: int) -> None:
    for p in _PROFILES.values():
        p.commit(step)


def commit_all_graph() -> None:
    for p in _PROFILES.values():
        p.commit_graph()


def reset() -> None:
    for p in _PROFILES.values():
        p.detach()
    _PROFILES.clear()


__all__ = ["LayerProfile", "attach", "profile_of", "commit_all", "commit_all_graph", "reset", "get_hookable_modules", "LAYER_RECORD_DTYPE"]
