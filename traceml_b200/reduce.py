"""Cross-rank window reduce: the GPU-native final-summary path.

Replaces, for the Step-Time / Step-Memory / Process sections, the reference's
TCP -> SQLite -> single-core Python chain
(``src/traceml/reporting/sections/*/loader.py`` + ``diagnostics/*``): every
rank's window stays resident in its own HBM ring; ranks agree on the common
step window with one or two tiny collectives, exchange their aligned 64-B rows
once over NVLink (peer loads fused into the reduce kernel, a step-sharded
send/recv, or one NCCL all-gather), and each GPU reduces its shard of the steps.

Two drivers sequence the same C-ABI stages:
  * production (one engine per process on a CUDA device): ``tml_reduce_run``
    (``csrc/tml_summary.cpp``) runs stages and NCCL collectives natively on
    torch.distributed's own communicator -- ``WindowReducer.run_native``;
  * this module's Python staging: several engines per process ("local ranks":
    how single-GPU tests play a whole job on one device), gloo on CPU, or when the
    communicator cannot be borrowed.  It is also the executable specification of
    the native driver; the two are held bit-identical by the tests.

All per-step arithmetic is in ``csrc/tml_engine.cu``, all rank-level rules in
``csrc/tml_diag.cpp``.  Both drivers fill the same ``_abi.ReduceRunOut`` as they go, which
``csrc/tml_sections.cpp`` turns into sections, and both return it in one view, ``ReduceResult``.
"""

from __future__ import annotations

import functools
import math
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from . import _abi

KIND_TIME, KIND_MEM = _abi.KIND_TIME, _abi.KIND_MEM

_INFO_LEN = 23
_ALIGN_LEN = 15 + 72  # sums + the 72-byte CUDA-IPC rows handle, one byte per double
_PROC_FIELDS = tuple(f for f, _ in _abi.ProcAgg._fields_)
_PROC_INT_FIELDS = ("n", "n_gpu", "max_cores", "any_gpu_available")
_PROC_U64_FIELDS = ("sum_rss", "sum_used", "sum_resv")  # exact byte sums: two 32-bit halves each
_PROC_LEN = len(_PROC_FIELDS) + len(_PROC_U64_FIELDS)


def _proc_pack(a) -> List[float]:
    """A ``ProcAgg`` as doubles for the exchange (csrc/tml_summary.cpp pack_proc: same layout).
    The u64 byte sums go as low and high 32-bit halves, each exact in a double."""
    v: List[float] = []
    for f in _PROC_FIELDS:
        x = getattr(a, f)
        if f in _PROC_U64_FIELDS:
            v.extend((float(x & 0xFFFFFFFF), float(x >> 32)))
        else:
            v.append(float(x))
    return v


def _proc_unpack(v, a) -> None:
    """The inverse of ``_proc_pack``, into the ``ProcAgg`` ``a``."""
    k = 0
    for f in _PROC_FIELDS:
        if f in _PROC_U64_FIELDS:
            setattr(a, f, int(v[k]) | (int(v[k + 1]) << 32))
            k += 2
        else:
            setattr(a, f, int(round(v[k])) if f in _PROC_INT_FIELDS else v[k])
            k += 1

# analytics/trends/schema.py:27-62
_BANDS = ((0.15, 0.25), (0.45, 0.55), (0.90, 1.00))
_HISTORY_LIMIT = 10_000


# ----------------------------------------------------------------------------- comm
class LocalComm:
    """Single process: every collective is the identity."""

    world = 1
    index = 0

    def all_gather_vec(self, vec, device=None) -> List[List[float]]:
        return [list(vec)]

    def all_reduce_min_(self, t: torch.Tensor) -> None:
        return None

    def all_gather_into(self, out: torch.Tensor, inp: torch.Tensor) -> None:
        out.copy_(inp)

    def all_to_all(self, out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits) -> None:
        out.copy_(inp)

    def barrier(self) -> None:
        return None

    def nccl_comm_ptr(self, device) -> Optional[int]:
        return None

    def one_host(self, device=None) -> bool:
        return True


class TorchDistComm:
    """torch.distributed plumbing (NCCL over NVLink on the box, gloo in CPU tests)."""

    def __init__(self, group=None):
        import torch.distributed as dist

        self._dist = dist
        self.group = group
        self.n_vec = 0  # small vector all-gathers issued (the latency-bound exchanges)
        self._comm_ptr: Optional[int] = None
        self._one_host: Optional[bool] = None
        self.world = dist.get_world_size(group)
        self.index = dist.get_rank(group)

    def one_host(self, device=None) -> bool:
        """Do all ranks of the group run on this host?  CUDA-IPC peer mappings (the ``p2p`` row
        exchange) exist only between processes of one host.  Collective on its first call (one
        all-gather of a 48-bit host-name hash), cached afterwards."""
        if self._one_host is None:
            if self.world == 1:
                self._one_host = True
            else:
                import hashlib
                import socket

                h = int.from_bytes(hashlib.blake2b(socket.gethostname().encode(), digest_size=6).digest(), "big")
                dev = device or torch.device("cpu")
                inp = torch.tensor([float(h)], dtype=torch.float64, device=dev)  # < 2^48: exact in f64
                out = torch.empty(self.world, dtype=torch.float64, device=dev)
                self._dist.all_gather_into_tensor(out, inp, group=self.group)
                self._one_host = bool((out == out[0]).all().item())
        return self._one_host

    def nccl_comm_ptr(self, device: torch.device) -> Optional[int]:
        """The ncclComm_t torch.distributed already holds for this group and device (the
        native reduce issues its collectives on it); None when there is none to borrow."""
        if self._comm_ptr is not None:
            return self._comm_ptr or None
        self._comm_ptr = 0
        try:
            if device.type == "cuda" and self._dist.get_backend(self.group) == "nccl":
                pg = self.group or self._dist.distributed_c10d._get_default_group()
                be = pg._get_backend(device)
                if not be._is_initialized():  # lazy communicator: one tiny collective creates it
                    self._dist.all_reduce(torch.zeros(1, device=device), group=self.group)
                    torch.cuda.synchronize(device)
                self._comm_ptr = int(be._comm_ptr())
        except Exception:  # noqa: BLE001 -- private torch API: fall back to the torch collectives
            self._comm_ptr = 0
        return self._comm_ptr or None

    def all_gather_vec(self, vec, device=None) -> List[List[float]]:
        """Fixed-length f64 vectors: one small all-gather, no pickling."""
        self.n_vec += 1
        dev = device or torch.device("cpu")
        inp = torch.tensor(list(vec), dtype=torch.float64, device=dev)
        out = torch.empty(self.world * inp.numel(), dtype=torch.float64, device=dev)
        self._dist.all_gather_into_tensor(out, inp, group=self.group)
        return out.view(self.world, -1).cpu().tolist()

    def all_reduce_min_(self, t: torch.Tensor) -> None:
        self._dist.all_reduce(t, op=self._dist.ReduceOp.MIN, group=self.group)

    def all_gather_into(self, out: torch.Tensor, inp: torch.Tensor) -> None:
        self._dist.all_gather_into_tensor(out, inp, group=self.group)

    def all_to_all(self, out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits) -> None:
        self._dist.all_to_all_single(out, inp, list(out_splits), list(in_splits), group=self.group)

    def barrier(self) -> None:
        self._dist.barrier(group=self.group)


# ----------------------------------------------------------------------------- helpers
def _band_bounds(n: int, band) -> tuple:
    """analytics/trends/core.py:38-49."""
    start = int(math.floor(n * float(band[0])))
    end = int(math.ceil(n * float(band[1])))
    start = max(0, min(start, n - 1))
    end = max(start + 1, min(end, n))
    return start, end


def trend_layout(n: int, *, min_points: int, warmup_frac: float):
    """Global series index ranges of the three trend bands, or None if the
    series is too short (analytics/trends/core.py:51-84).  csrc/tml_summary.cpp:trend_layout is the
    native driver's copy: tests/test_gpu_align_bands.py::test_build_band_layout keeps both equal to
    the oracle's bands."""
    if n < min_points:
        return None
    length = min(n, _HISTORY_LIMIT)
    if length < min_points:
        return None
    off = n - length
    warm = int(math.floor(length * float(warmup_frac)))
    stable = length - warm
    if stable < min_points:
        return None
    out = []
    for b in _BANDS:
        s, e = _band_bounds(stable, b)
        out.append((off + warm + s, off + warm + e))
    return out


def _stream_of(device: torch.device) -> int:
    """The raw handle of ``device``'s current stream (0 off CUDA), without a ``torch.cuda.Stream``."""
    if device.type != "cuda":
        return 0
    index = device.index if device.index is not None else torch.cuda.current_device()
    return torch._C._cuda_getCurrentRawStream(index)


class ReduceKind:
    """One section of a ``ReduceResult``: ``series`` is this process's [16, n_common] (its
    ``shard`` of the columns valid), None without a reduce pass.  Every other field (alignment,
    bands) is read from the section's ``KindResultC`` in ``ReduceResult.out``."""

    def __init__(self, k, series: Optional[torch.Tensor]):
        self._k = k
        self.n_common = int(k.n_common)
        self.shard = (int(k.shard_lo), int(k.shard_hi))
        self.series = series

    def __getattr__(self, name: str):
        return getattr(self.__dict__["_k"], name)


class ReduceResult:
    """One reduce's result, whichever driver sequenced it: ``out``, the ``_abi.ReduceRunOut`` the
    section emitter reads (per-rank infos and process aggregates, the alignment and bands of
    ``out.time`` / ``out.mem``), and the facts callers read from it.

    ``exchange`` names the row exchange used; ``timings_ms`` holds the driver's stage times.
    ``series``: the series tensors the Python driver wrote, by kind; without them (native
    driver) ``time.series`` / ``mem.series`` are zero-copy, read-only views of the engine's own
    workspace: valid until the engine's next reduce or its ``close()``; ``clone()`` them to keep
    them.  Their row stride may exceed ``n_common``, and when ``series_paired`` is set (the
    single-rank bulk path) rows 2m and 2m+1 are the same memory mapped twice, so a write into one
    row would change its partner."""

    def __init__(self, out: _abi.ReduceRunOut, window: int, exchange: str, timings_ms: Dict[str, float],
                 series: Optional[Dict[str, Optional[torch.Tensor]]] = None,
                 device: Optional[torch.device] = None):
        self.out = out
        self.window = window
        self.exchange = exchange
        self.timings_ms = timings_ms
        self._series = series
        self._device = device

    ranks = property(lambda self: list(range(int(self.out.n_ranks))))
    fused_pass = property(lambda self: bool(self.out.fused_pass))
    fused_rows = property(lambda self: int(self.out.fused_pass) == 2)  # single-rank bulk: ring -> series in one kernel
    series_paired = property(lambda self: bool(self.out.time.series_paired))
    n_exchanges = property(lambda self: int(self.out.n_exchanges))

    @functools.cached_property
    def time(self) -> ReduceKind:
        return self._kind("time")

    @functools.cached_property
    def mem(self) -> ReduceKind:
        return self._kind("mem")

    @property
    def proc_aggs(self) -> Dict[int, Dict[str, Any]]:
        """Every rank's process aggregates (``out.procs``) as dicts of their fields; zeros when the
        reduce had no process rows."""
        return {r: {f: getattr(self.out.procs[r], f) for f in _PROC_FIELDS} for r in self.ranks}

    def _kind(self, name: str) -> ReduceKind:
        k = getattr(self.out, name)
        n = int(k.n_common)
        if self._series is not None:
            series = self._series.get(name)
        elif k.series and n:
            from .engine import _DevView

            ld = int(k.series_ld)
            series = torch.as_tensor(_DevView(int(k.series), _abi.TML_SERIES_PER_STEP * ld),
                                     device=self._device).view(_abi.TML_SERIES_PER_STEP, ld)[:, :n]
        else:
            series = None
        return ReduceKind(k, series)

    def __reduce__(self):
        """Pickles as the bytes of ``out`` and what the Python driver kept.  ctypes cannot pickle
        ``out`` itself (it has pointer fields), and the series pointers mean nothing in another
        process: they travel zeroed, so the native driver's series views do not travel."""
        o = type(self.out).from_buffer_copy(self.out)
        o.time.series = o.mem.series = None
        return (_result_restore, (bytes(o), self.window, self.exchange, self.timings_ms, self._series))


def _result_restore(raw, window, exchange, timings_ms, series) -> ReduceResult:
    return ReduceResult(_abi.ReduceRunOut.from_buffer_copy(raw), window, exchange, timings_ms, series)


# ----------------------------------------------------------------------------- reducer
class WindowReducer:
    """Sequences the reduce stages for the local engines of this process."""

    def __init__(self, engines: Sequence[Any], comm: Any = None, *, device: Optional[torch.device] = None,
                 exchange: str = "auto", speculate: bool = True, native: bool = True):
        self.speculate = speculate
        self.native = native        # False: sequence the stages from Python (reference driver)
        self.engines = list(engines)
        self.comm = comm or LocalComm()
        self.device = device or torch.device("cuda", self.engines[0].device)
        self.L = len(self.engines)
        self.exchange = exchange
        self._p2p_warm = False  # peer mappings already open: p2p costs nothing extra
        self._k4_events: List[Any] = []

    def _peers_on_this_host(self) -> bool:
        """CUDA-IPC (p2p) is possible: every rank of the group is a process of this host."""
        fn = getattr(self.comm, "one_host", None)
        return True if fn is None else bool(fn(self.device))

    # global rank of local engine l
    def _grank(self, l: int) -> int:
        return self.comm.index * self.L + l

    @staticmethod
    def _info_pack(w, mem: Tuple[int, int]) -> List[float]:
        """A rank's ``WinInfo`` as doubles for the exchange (csrc/tml_summary.cpp pack_info: same
        layout), advertising ``mem`` = (lo, n_cand) for its memory candidates."""
        lo, n_cand = list(w.lo), list(w.n_cand)
        lo[KIND_MEM], n_cand[KIND_MEM] = mem
        return ([w.n_retained, w.latest_step, w.monotone, w.dup_rows] + list(w.n_rows) + n_cand + lo
                + list(w.hi) + list(w.t_sums) + [w.t_count, w.n_both] + list(w.dense))

    @staticmethod
    def _info_unpack(v: Sequence[float], i) -> None:
        """The inverse of ``_info_pack``, into the ``WinInfo`` ``i``."""
        n = lambda x: int(round(x))  # noqa: E731  (step ids < 2^53)
        i.n_retained, i.latest_step, i.monotone, i.dup_rows = (n(x) for x in v[0:4])
        for q in range(2):
            i.n_rows[q], i.n_cand[q], i.lo[q], i.hi[q] = n(v[4 + q]), n(v[6 + q]), n(v[8 + q]), n(v[10 + q])
            i.dense[q] = n(v[21 + q])
        i.t_sums[:] = [float(x) for x in v[12:19]]
        i.t_count, i.n_both = n(v[19]), n(v[20])

    def reduce(self, window: int, *, proc_rows: Optional[int] = None, stage_timings: bool = False) -> ReduceResult:
        """``stage_timings``: per-stage CUDA-event / host-clock breakdown (a diagnostic: a dozen torch
        events per call).  Without it ``timings_ms`` still carries ``k3a`` / ``k4``, the
        two kernels' device times from the library's own events.

        The Python staging fills its ``ReduceRunOut`` the way ``reduce_run`` in
        csrc/tml_summary.cpp fills ``out``, except for the exchange code and the native driver's
        counters and times, which stay zero."""
        window = max(1, int(window))
        dev = self.device
        stream = _stream_of(dev)
        if self._native_ok() and not stage_timings:
            return self.native_result(self.run_native(window, proc_rows, stream), window)
        self._k4_events = []
        self._timed = bool(stage_timings)
        R = self.comm.world * self.L
        o = _abi.ReduceRunOut()
        o.n_ranks = R
        ev = None
        timings: Dict[str, float] = {}
        import time as _time

        hw = [_time.perf_counter()]
        if stage_timings and dev.type == "cuda":
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
            ev[0].record()

        # ---- stage 1: local windows + bounds
        if proc_rows:  # K6 first, un-synchronised: win_prepare's sync below covers it
            for e in self.engines:
                if hasattr(e, "proc_reduce_launch"):
                    e.proc_reduce_launch(max(1, int(proc_rows)), stream)
        k3a_ev = k3a_ev0 = None
        if ev:
            k3a_ev0 = torch.cuda.Event(enable_timing=True)
            k3a_ev0.record()
        local = [e.win_prepare(window, stream) for e in self.engines]
        if ev:
            k3a_ev = torch.cuda.Event(enable_timing=True)
            k3a_ev.record()
        mems = [self._memory_candidates(e, w, window, stream) for e, w in zip(self.engines, local)]
        # Lock-step speculation: a rank whose own time window is dense assumes the common
        # window IS its window (true whenever the ranks run in lock step) and sends that
        # alignment -- sums and rows handle, nothing to launch -- with its bounds.  If the
        # gathered bounds confirm it, the separate alignment exchange is skipped.
        plen = _PROC_LEN if proc_rows else 0
        slen = self._spec_len()
        per = _INFO_LEN + plen + slen
        flat: List[float] = []
        for eng, w, mem in zip(self.engines, local, mems):
            flat.extend(self._info_pack(w, mem))
            if proc_rows:  # process aggregates (K6) ride in the same exchange
                a = (eng.proc_reduce_collect() if hasattr(eng, "proc_reduce_collect")
                     else eng.proc_reduce(max(1, int(proc_rows)), stream))
                flat.extend(_proc_pack(a))
            if slen:
                sp = [0.0] * slen
                if w.dense[KIND_TIME] and w.n_cand[KIND_TIME] > 0:
                    a = eng.win_select_dense(KIND_TIME, w.lo[KIND_TIME], w.n_cand[KIND_TIME], stream)
                    sp = self._align_pack(eng, KIND_TIME, a, slen)
                flat.extend(sp)
        spec: Optional[List[List[float]]] = [] if slen else None
        for p, row in enumerate(self.comm.all_gather_vec(flat, dev)):
            srow: List[float] = []
            for l in range(self.L):
                v = row[l * per:(l + 1) * per]
                self._info_unpack(v[:_INFO_LEN], o.infos[p * self.L + l])
                if proc_rows:
                    _proc_unpack(v[_INFO_LEN:_INFO_LEN + plen], o.procs[p * self.L + l])
                srow.extend(v[_INFO_LEN + plen:])
            if spec is not None:
                spec.append(srow)
        hw.append(_time.perf_counter())
        if ev:
            ev[1].record()

        # If on every rank the time and the memory candidates are the very same rows (the
        # common case: ring not longer than the window, every step has memory), one
        # alignment serves both sections.
        t, m = o.time, o.mem
        merged = all(i.n_cand[0] == i.n_cand[1] == i.n_both for i in o.infos[:R])
        t_handles = self._align(KIND_TIME, window, o.infos, R, t, stream, spec=spec)
        if merged:
            o.mem = o.time  # a copy, of the alignment: nothing else is set yet
            m_handles = t_handles
        else:
            m_handles = self._align(KIND_MEM, window, o.infos, R, m, stream)
        hw.append(_time.perf_counter())
        if ev:
            ev[2].record()

        # ---- stage 4: exchange + per-step reduce
        same = (t.n_common > 0 and t.n_common == m.n_common and t.start_step == m.start_step
                and t.end_step == m.end_step and t.used[:t.n_used] == m.used[:m.n_used])
        mode = self._exchange_mode(t.n_common or m.n_common)
        series: Dict[str, Optional[torch.Tensor]] = {"time": None, "mem": None}
        if same:
            series["time"] = series["mem"] = self._reduce_pass(
                KIND_TIME, _abi.MASK_TIME | _abi.MASK_MEM, t, t_handles, stream, mode)
            m.series, m.series_ld, m.shard_lo, m.shard_hi = t.series, t.series_ld, t.shard_lo, t.shard_hi
        else:
            if t.n_common:
                series["time"] = self._reduce_pass(KIND_TIME, _abi.MASK_TIME, t, t_handles, stream,
                                                   self._exchange_mode(t.n_common))
            if m.n_common:
                series["mem"] = self._reduce_pass(KIND_MEM, _abi.MASK_MEM, m, m_handles, stream,
                                                  self._exchange_mode(m.n_common))
        o.fused_pass = 1 if same else 0
        if mode == "p2p":
            self._p2p_warm = True
        hw.append(_time.perf_counter())
        if ev:
            ev[3].record()

        # ---- stage 5: trend bands
        self._bands(t, series["time"], stream)
        if same:  # the memory section's series is the time section's: so are its bands
            m.has_bands, m.band_sum, m.band_cnt = t.has_bands, t.band_sum, t.band_cnt
            m.tail_first, m.tail_last = t.tail_first, t.tail_last
        else:
            self._bands(m, series["mem"], stream)
        hw.append(_time.perf_counter())
        for i, nm in enumerate(("prepare", "align", "reduce", "bands")):
            timings["host_" + nm] = (hw[i + 1] - hw[i]) * 1e3
        k3a = max((float(getattr(w, "kernel_ms", 0.0)) for w in local), default=0.0)
        if ev:
            ev[4].record()
            torch.cuda.synchronize(dev)
            names = ["prepare", "align", "reduce", "bands"]
            for i, nm in enumerate(names):
                timings[nm] = float(ev[i].elapsed_time(ev[i + 1]))
            timings["total"] = float(ev[0].elapsed_time(ev[4]))
            timings["k3a_stage"] = float(k3a_ev0.elapsed_time(k3a_ev))
            timings["k3a"] = k3a or timings["k3a_stage"]
            timings["k4"] = float(sum(a.elapsed_time(b) for a, b in self._k4_events))
        elif dev.type == "cuda":  # the bands stage synchronised: both kernels have finished
            timings["k3a"] = k3a
            if t.n_common or m.n_common:
                timings["k4"] = float(sum(max(0.0, e.kernel_ms(1)) for e in self.engines
                                          if hasattr(e, "kernel_ms")))
        return ReduceResult(o, window, mode, timings, series)

    # ------------------------------------------------------------------ memory candidate limit
    def _memory_candidates(self, engine, info, window: int, stream) -> Tuple[int, int]:
        """(lo, n_cand) of the memory candidates a rank advertises.  Only the newest
        ``max(20 W, W + 1)`` distinct step ids of a rank enter the memory alignment
        (step_memory/loader.py:215, oracle candidate_rows).  The ring normally holds 1.5 W rows,
        so this binds only for a small window over a long ring; then the rank advertises the step
        id of its limit-th newest candidate as its lower bound -- every later stage works on
        [max lo, min hi] and never sees the older candidates."""
        limit = max(20 * window, window + 1)
        lo, n_cand = int(info.lo[KIND_MEM]), int(info.n_cand[KIND_MEM])
        if n_cand <= limit:
            return lo, n_cand
        hi = int(info.hi[KIND_MEM])
        if info.dense[KIND_MEM]:  # consecutive ids
            return hi - limit + 1, limit
        # holes / re-flushed ids: select the newest `limit` of its own
        span = hi - lo + 1
        own = torch.empty(span, dtype=torch.uint8, device=self.device)
        engine.win_presence(KIND_MEM, lo, span, own, stream)
        return int(engine.win_select(KIND_MEM, lo, span, own, limit, stream).start_step), limit

    # ------------------------------------------------------------------ native sequencing
    def _native_ok(self) -> bool:
        """One rank per process on a CUDA device: csrc/tml_summary.cpp runs the stages and
        the collectives itself (on torch.distributed's own communicator)."""
        if not self.native or self.L != 1 or self.device.type != "cuda":
            return False
        if not hasattr(self.engines[0], "reduce_run") or self.exchange == "nccl":
            return False
        if self.comm.world == 1:
            return True
        return bool(getattr(self.comm, "nccl_comm_ptr", lambda d: None)(self.device))

    def run_native(self, window: int, proc_rows: Optional[int], stream: Optional[int] = None, prev=None,
                   out=None):
        """tml_reduce_run on this process's engine; the raw result struct: ``out`` if given, else the
        engine's own (valid until the next run).  ``prev``: see ``Engine.reduce_run``."""
        eng = self.engines[0]
        world = self.comm.world
        ptr = self.comm.nccl_comm_ptr(self.device) if world > 1 else 0
        xchg = self.exchange if self.exchange in _abi.XCHG else "auto"
        if xchg == "auto" and world > 1 and not self._peers_on_this_host():
            xchg = "a2a"  # the native driver's own "auto" assumes one host (p2p from 10^6 rows)
        return eng.reduce_run(window, int(proc_rows or 0), xchg,
                              self.speculate, ptr or 0, self.comm.index, world,
                              _stream_of(self.device) if stream is None else stream, prev=prev, out=out)

    @staticmethod
    def native_timings(o) -> Dict[str, float]:
        p, a, r, b, t = o.stage_ms[:]  # the stages end in a sync: host and device times are one
        return {"host_prepare": p, "host_align": a, "host_reduce": r, "host_bands": b, "host_total": t,
                "prepare": p, "align": a, "reduce": r, "bands": b, "total": t,
                "k3a": o.k3a_ms, "k4": max(0.0, o.k4_ms)}

    def native_result(self, o, window: int, *, owned: bool = False) -> ReduceResult:
        """The view of a ``run_native`` result: over ``o`` itself when the caller hands it over
        (``owned``, a struct no later run writes), else over its own copy, since the engine reuses
        its struct."""
        return ReduceResult(o if owned else type(o).from_buffer_copy(o), window,
                            _abi.XCHG_NAME[o.exchange_used], self.native_timings(o), device=self.device)

    # ------------------------------------------------------------------ alignment
    def _spec_len(self) -> int:
        """Length of the speculative alignment block in the first exchange (0 = off)."""
        if not self.speculate:
            return 0
        handles = self.comm.world > 1 and self.device.type == "cuda" and (
            self.exchange == "p2p" or (self.exchange == "auto" and self._peers_on_this_host()))
        return _ALIGN_LEN if handles else 15

    def _align(self, kind: int, window: int, infos, R: int, res, stream, spec=None) -> Dict[int, bytes]:
        """The alignment of ``kind`` over the ``R`` ranks' ``infos``, into ``res`` (a
        ``KindResultC``); the CUDA-IPC rows handle of every used rank (see ``_parse_aligns``)."""
        part = [r for r in range(R) if infos[r].n_cand[kind] > 0]
        res.observed = len(part)
        if not part:
            return {}
        glo = max(infos[r].lo[kind] for r in part)
        ghi = min(infos[r].hi[kind] for r in part)
        if ghi < glo:
            return {}
        span = ghi - glo + 1
        dev = self.device
        if all(infos[r].dense[kind] for r in part):
            if (spec is not None and span <= window
                    and all(infos[r].lo[kind] == glo and infos[r].hi[kind] == ghi for r in part)):
                # every participant speculated on exactly [glo, ghi]: its block is the alignment
                return self._parse_aligns(res, spec, self._spec_len(), part)
            # lock-step fast path: every participant holds every step id of [glo, ghi]
            n_common = min(span, window)
            first = ghi - n_common + 1
            flat: List[float] = []
            for l, e in enumerate(self.engines):
                a = e.win_select_dense(kind, first, n_common, stream)
                flat.extend(self._align_pack(e, kind, a))
            return self._collect_aligns(res, flat, part)
        presence = None
        for l, e in enumerate(self.engines):
            p = torch.empty(span, dtype=torch.uint8, device=dev)
            e.win_presence(kind, glo, span, p, stream)
            presence = p if presence is None else torch.minimum(presence, p)
        self.comm.all_reduce_min_(presence)
        flat = []
        for l, e in enumerate(self.engines):
            a = e.win_select(kind, glo, span, presence, window, stream)
            flat.extend(self._align_pack(e, kind, a))
        return self._collect_aligns(res, flat, part)

    def _align_pack(self, engine, kind, a, length: Optional[int] = None) -> List[float]:
        """15 numbers + (p2p only) the rows' CUDA-IPC handle, so the peer mapping
        needs no collective of its own.  ``length`` fixes the block size (speculative
        block: every rank must send the same layout before n_common is agreed)."""
        out = ([int(a.n_common), int(a.start_step), int(a.end_step), int(a.n_rows)]
               + [float(x) for x in a.t_sums] + [float(x) for x in a.m_sums])
        p2p = self._exchange_mode(int(a.n_common)) == "p2p"
        if p2p and (length is None or length == _ALIGN_LEN):
            handle = engine.win_rows_export(kind) if int(a.n_rows) > 0 else bytes(72)
            out += [float(b) for b in handle]
        if length is not None:
            out += [0.0] * (length - len(out))
        return out

    def _collect_aligns(self, res, flat, part) -> Dict[int, bytes]:
        # n_common is identical on every rank, so every rank packed the same layout
        alen = _ALIGN_LEN if len(flat) == _ALIGN_LEN * self.L else 15
        return self._parse_aligns(res, self.comm.all_gather_vec(flat, self.device), alen, part)

    def _parse_aligns(self, res, rows, alen, part) -> Dict[int, bytes]:
        """``res``'s alignment from the gathered blocks, ``alen`` numbers per rank: the ranks of
        ``part`` with aligned rows, in ascending order.  Returns their rows handles (empty unless
        the blocks carry them: p2p)."""
        i = lambda x: int(round(x))  # noqa: E731
        blocks = [row[l * alen:(l + 1) * alen] for row in rows for l in range(self.L)]  # by global rank
        res.n_common = max(i(v[0]) for v in blocks)
        handles: Dict[int, bytes] = {}
        if res.n_common == 0:
            return handles
        for r, v in enumerate(blocks):
            if r in part and i(v[3]) > 0:
                u = res.n_used
                res.used[u], res.n_rows[u] = r, i(v[3])
                res.t_sums[u][:], res.m_sums[u][:] = list(v[4:11]), list(v[11:15])
                res.start_step, res.end_step = i(v[1]), i(v[2])
                res.n_used = u + 1
                handles[r] = bytes(i(b) for b in v[15:87]) if alen == _ALIGN_LEN else b""
        return handles

    # ------------------------------------------------------------------ exchange
    # One-shot cost of the fused peer-load exchange is the CUDA-IPC mapping of R-1 peer
    # allocations (tens of ms the first time, 0 once cached), so it
    # pays only for large or repeated windows.  Below this many aligned rows per rank the
    # step-sharded NCCL all-to-all is the default.
    P2P_MIN_ROWS = 1_000_000

    def _exchange_mode(self, n_common: Optional[int] = None) -> str:
        if self.comm.world == 1:
            return "local"
        if self.exchange in ("p2p", "nccl", "a2a"):
            if self.exchange == "a2a" and self.L != 1:
                return "nccl"
            return self.exchange
        if self.device.type != "cuda":
            return "nccl"
        if n_common is not None and n_common < self.P2P_MIN_ROWS and not self._p2p_warm:
            return "a2a" if self.L == 1 else "nccl"
        if not self._peers_on_this_host():  # ranks on other hosts: no peer mappings to load through
            return "a2a" if self.L == 1 else "nccl"
        return "p2p"

    def _reduce_pass(self, kind: int, mask: int, res, handles: Dict[int, bytes], stream,
                     mode: str) -> torch.Tensor:
        """The per-step series of ``res``'s aligned window, over the row exchange ``mode``: fills
        ``res``'s series fields and returns the [16, n_common] tensor they point into."""
        n = res.n_common
        used = res.used[:res.n_used]
        dev = self.device
        # series buffer of this process: [16, n]; only this process's shard is written
        series = torch.empty(_abi.TML_SERIES_PER_STEP * n, dtype=torch.float64, device=dev)
        my = [self._grank(l) for l in range(self.L)]
        # rows handle per used rank
        rows: Dict[int, Any] = {}
        if mode == "local":
            for r in used:
                rows[r] = self.engines[r - self.comm.index * self.L].win_rows_tensor(kind, n)
        elif mode == "nccl":
            # one all-gather of the dense aligned rows; ranks outside `used` send zeros
            W = self.comm.world * self.L
            gathered = torch.empty(W * n * 8, dtype=torch.float64, device=dev)
            local = torch.zeros(self.L * n * 8, dtype=torch.float64, device=dev)
            for l in range(self.L):
                if self._grank(l) in used:
                    local[l * n * 8:(l + 1) * n * 8].copy_(self.engines[l].win_rows_tensor(kind, n))
            self.comm.all_gather_into(gathered, local)
            for r in used:
                rows[r] = gathered[r * n * 8:(r + 1) * n * 8]
            self._keep = gathered
        elif mode == "a2a":
            # step-sharded NCCL all-to-all: rank g receives only the rows of ITS shard of the
            # steps from every rank ((R-1)/R * n * 64 B instead of (R-1) * n * 64 B), and K4
            # reads them through virtual base pointers (row j of rank r sits at
            # recv[r] + (j - shard_lo) * 64)
            W = self.comm.world
            g = self.comm.index
            bounds = [(n * d) // W for d in range(W + 1)]
            mine = (self.engines[0].win_rows_tensor(kind, n) if g in used
                    else torch.zeros(n * 8, dtype=torch.float64, device=dev))
            my_len = bounds[g + 1] - bounds[g]
            recv = torch.empty(max(1, W * my_len * 8), dtype=torch.float64, device=dev)
            self.comm.all_to_all(recv[:W * my_len * 8], mine, [my_len * 8] * W,
                                 [(bounds[d + 1] - bounds[d]) * 8 for d in range(W)])
            for r in used:
                rows[r] = recv.data_ptr() + (r * my_len - bounds[g]) * 64
            self._keep = recv
        else:
            # p2p: CUDA-IPC peer mappings, loads fused into the reduce kernel.  No barrier is
            # needed around it: (1) a rank's rows are complete before it enters the aligns
            # all-gather (win_select* synchronises its stream), so once that collective
            # returns every peer's rows are readable; (2) a rank overwrites its rows only in
            # the NEXT reduce's win_prepare, which comes after this reduce's band all-gather,
            # and every rank enters that only after its own K4 has finished (win_bands syncs).
            e0 = self.engines[0]
            for r in used:
                if r in my:
                    rows[r] = self.engines[r - self.comm.index * self.L].win_rows_tensor(kind, n)
                else:
                    rows[r] = e0.peer_open(handles[r])
        # step-sharded: shard s of W_total shards -> engine with global rank s
        W = self.comm.world * self.L
        lo_first, hi_last = None, None
        timed = self._timed and self.device.type == "cuda"
        if timed:
            k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            k0.record()
        for l, e in enumerate(self.engines):
            g = self._grank(l)
            lo = (n * g) // W
            hi = (n * (g + 1)) // W
            if lo_first is None:
                lo_first = lo
            hi_last = hi
            if hi > lo:
                e.win_reduce([rows[r] for r in used], mask, n, lo, hi, series, stream)
        if timed:
            k1.record()
            self._k4_events.append((k0, k1))
        res.series, res.series_ld = series.data_ptr(), n
        res.shard_lo, res.shard_hi = lo_first or 0, hi_last or 0
        return series.view(_abi.TML_SERIES_PER_STEP, n)

    # ------------------------------------------------------------------ bands
    def _bands(self, res, series: Optional[torch.Tensor], stream) -> None:
        """``res``'s trend bands from this process's shard of ``series``, summed over the ranks."""
        n = res.n_common
        if n == 0 or series is None:
            return
        a = _abi.BandArgs()
        a.n_common = n
        a.shard_lo, a.shard_hi = res.shard_lo, res.shard_hi
        lay_t = trend_layout(n, min_points=200, warmup_frac=0.10)
        lay_m = trend_layout(n, min_points=50, warmup_frac=0.0)
        for k, lay in ((0, lay_t), (1, lay_m)):
            for b in range(3):
                a.band_lo[k][b] = lay[b][0] if lay else 0
                a.band_hi[k][b] = lay[b][1] if lay else 0
        a.tail_first[0] = 0
        a.tail_first[1] = n - min(n, 1000)
        out = self.engines[0].win_bands(series, a, stream)
        vec = ([float(out.sum[s][b]) for s in range(16) for b in range(3)]
               + [float(out.cnt[s][b]) for s in range(16) for b in range(3)]
               + [float(out.tail_first[s]) for s in range(16)]
               + [float(out.tail_last[s]) for s in range(16)])
        rows = self.comm.all_gather_vec(vec, self.device)
        for s in range(16):
            for b in range(3):  # sums in rank order
                res.band_sum[s][b] = sum(row[s * 3 + b] for row in rows)
                res.band_cnt[s][b] = sum(int(round(row[48 + s * 3 + b])) for row in rows)
            # the tails come from the one rank whose shard holds their step
            res.tail_first[s] = next((row[96 + s] for row in rows if not math.isnan(row[96 + s])), math.nan)
            res.tail_last[s] = next((row[112 + s] for row in rows if not math.isnan(row[112 + s])), math.nan)
        res.has_bands = 1


__all__ = ["WindowReducer", "LocalComm", "TorchDistComm", "ReduceResult", "ReduceKind", "trend_layout"]
