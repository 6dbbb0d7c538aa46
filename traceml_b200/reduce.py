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
``csrc/tml_diag.cpp``.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence

import torch

from . import _abi

KIND_TIME, KIND_MEM = _abi.KIND_TIME, _abi.KIND_MEM

_INFO_LEN = 23
_ALIGN_LEN = 15 + 72  # sums + the 72-byte CUDA-IPC rows handle, one byte per double
_PROC_FIELDS = tuple(f for f, _ in _abi.ProcAgg._fields_)
_PROC_INT_FIELDS = ("n", "n_gpu", "max_cores", "any_gpu_available")
_PROC_LEN = len(_PROC_FIELDS)

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
    series is too short (analytics/trends/core.py:51-84)."""
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
    return int(torch.cuda.current_stream(device).cuda_stream) if device.type == "cuda" else 0


@dataclass
class RankWindow:
    """What one global rank contributed to one aligned window."""

    rank: int
    n_rows: int = 0
    t_sums: Sequence[float] = ()
    m_sums: Sequence[float] = ()
    info: Dict[str, Any] = field(default_factory=dict)


@dataclass
class KindResult:
    observed: int = 0            # ranks that had candidates
    used: List[int] = field(default_factory=list)
    n_common: int = 0
    start_step: Optional[int] = None
    end_step: Optional[int] = None
    windows: Dict[int, RankWindow] = field(default_factory=dict)
    band_sum: Optional[List[List[float]]] = None   # [16][3]
    band_cnt: Optional[List[List[int]]] = None
    tail_first: Optional[List[float]] = None
    tail_last: Optional[List[float]] = None
    series: Optional[torch.Tensor] = None          # this process's [16, n_common] (own shard valid)
    shard: tuple = (0, 0)


@dataclass
class ReduceOutput:
    window: int
    ranks: List[int]
    infos: Dict[int, Dict[str, Any]]
    time: KindResult
    mem: KindResult
    exchange: str
    fused_pass: bool
    timings_ms: Dict[str, float] = field(default_factory=dict)
    proc_aggs: Dict[int, Dict[str, Any]] = field(default_factory=dict)


class NativeReduceOutput:
    """What ``SummaryEngine.build`` returns as ``"reduce"`` on the native path: the cheap
    facts eagerly, the full ``ReduceOutput`` (per-rank windows, band sums, series view) only
    if somebody asks -- the sections no longer need it.  ``time.series`` / ``mem.series`` are
    zero-copy views of the engine's own workspace: valid until the engine's next reduce or its
    ``close()``; ``clone()`` them to keep them."""

    def __init__(self, reducer: "WindowReducer", o, window: int, proc_rows: Optional[int]):
        self.window = window
        self.exchange = _abi.XCHG_NAME[int(o.exchange_used)]
        self.fused_pass = bool(o.fused_pass)
        self.fused_rows = int(o.fused_pass) == 2  # single-rank bulk path: ring -> series in one kernel
        self.timings_ms = reducer.native_timings(o)
        self.n_exchanges = int(o.n_exchanges)
        self.ranks = list(range(int(o.n_ranks)))
        self._snap = type(o).from_buffer_copy(o)  # the engine reuses its result struct
        self._args = (reducer, window, proc_rows)
        self._full: Optional[ReduceOutput] = None

    def _get(self) -> ReduceOutput:
        if self._full is None:
            reducer, window, proc_rows = self._args
            self._full = reducer.convert_native(self._snap, window, proc_rows)
        return self._full

    time = property(lambda self: self._get().time)
    mem = property(lambda self: self._get().mem)
    infos = property(lambda self: self._get().infos)
    proc_aggs = property(lambda self: self._get().proc_aggs)


# ----------------------------------------------------------------------------- reducer
class WindowReducer:
    """Sequences the reduce stages for the local engines of this process."""

    def __init__(self, engines: Sequence[Any], comm: Any = None, *, device: Optional[torch.device] = None,
                 exchange: str = "auto", speculate: bool = True, native: bool = True):
        self.speculate = speculate
        self.native = native        # False: sequence the stages from Python (reference driver)
        self.last_exchanges = 0
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

    def _info_dict(self, w) -> Dict[str, Any]:
        return {
            "n_retained": int(w.n_retained), "latest_step": int(w.latest_step),
            "monotone": int(w.monotone), "dup_rows": int(w.dup_rows),
            "n_rows": [int(w.n_rows[0]), int(w.n_rows[1])],
            "n_cand": [int(w.n_cand[0]), int(w.n_cand[1])],
            "lo": [int(w.lo[0]), int(w.lo[1])], "hi": [int(w.hi[0]), int(w.hi[1])],
            "t_sums": [float(x) for x in w.t_sums], "t_count": int(w.t_count),
            "n_both": int(getattr(w, "n_both", 0)),
            "dense": [int(x) for x in getattr(w, "dense", (0, 0))],
            "kernel_ms": float(getattr(w, "kernel_ms", 0.0)),
        }

    @staticmethod
    def _info_pack(d: Dict[str, Any]) -> List[float]:
        return ([d["n_retained"], d["latest_step"], d["monotone"], d["dup_rows"]]
                + d["n_rows"] + d["n_cand"] + d["lo"] + d["hi"] + d["t_sums"] + [d["t_count"], d["n_both"]] + d["dense"])

    @staticmethod
    def _info_unpack(v: Sequence[float]) -> Dict[str, Any]:
        i = lambda x: int(round(x))  # noqa: E731  (step ids < 2^53)
        return {"n_retained": i(v[0]), "latest_step": i(v[1]), "monotone": i(v[2]),
                "dup_rows": i(v[3]), "n_rows": [i(v[4]), i(v[5])], "n_cand": [i(v[6]), i(v[7])],
                "lo": [i(v[8]), i(v[9])], "hi": [i(v[10]), i(v[11])],
                "t_sums": [float(x) for x in v[12:19]], "t_count": i(v[19]), "n_both": i(v[20]), "dense": [i(v[21]), i(v[22])]}

    def reduce(self, window: int, *, proc_rows: Optional[int] = None, overlap=None, stage_timings: bool = False) -> ReduceOutput:
        """``overlap(proc_aggs)``: host work that needs only the process aggregates; it
        runs after K4 has been launched and before the first wait on it.
        ``stage_timings``: per-stage CUDA-event / host-clock breakdown (a diagnostic: a dozen torch
        events per call).  Without it ``timings_ms`` still carries ``k3a`` / ``k4``, the
        two kernels' device times from the library's own events."""
        window = max(1, int(window))
        dev = self.device
        stream = _stream_of(dev)
        if self._native_ok() and not stage_timings:
            return self._reduce_native(window, proc_rows, stream)
        self._k4_events = []
        self._timed = bool(stage_timings)
        R = self.comm.world * self.L
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
        local_infos = [self._info_dict(e.win_prepare(window, stream)) for e in self.engines]
        if ev:
            k3a_ev = torch.cuda.Event(enable_timing=True)
            k3a_ev.record()
        for l, e in enumerate(self.engines):
            self._limit_memory_candidates(e, local_infos[l], window, stream)
        # Lock-step speculation: a rank whose own time window is dense assumes the common
        # window IS its window (true whenever the ranks run in lock step) and sends that
        # alignment -- sums and rows handle, nothing to launch -- with its bounds.  If the
        # gathered bounds confirm it, the separate alignment exchange is skipped.
        plen = _PROC_LEN if proc_rows else 0
        slen = self._spec_len()
        per = _INFO_LEN + plen + slen
        flat: List[float] = []
        for l, d in enumerate(local_infos):
            flat.extend(self._info_pack(d))
            eng = self.engines[l]
            if proc_rows:  # process aggregates (K6) ride in the same exchange
                a = (eng.proc_reduce_collect() if hasattr(eng, "proc_reduce_collect")
                     else eng.proc_reduce(max(1, int(proc_rows)), stream))
                flat.extend(float(getattr(a, f)) for f in _PROC_FIELDS)
            if slen:
                sp = [0.0] * slen
                if d["dense"][KIND_TIME] and d["n_cand"][KIND_TIME] > 0:
                    a = eng.win_select_dense(KIND_TIME, d["lo"][KIND_TIME], d["n_cand"][KIND_TIME], stream)
                    sp = self._align_pack(eng, KIND_TIME, a, slen)
                flat.extend(sp)
        infos: Dict[int, Dict[str, Any]] = {}
        proc_aggs: Dict[int, Dict[str, Any]] = {}
        spec: Optional[List[List[float]]] = [] if slen else None
        for p, row in enumerate(self.comm.all_gather_vec(flat, dev)):
            srow: List[float] = []
            for l in range(self.L):
                v = row[l * per:(l + 1) * per]
                infos[p * self.L + l] = self._info_unpack(v[:_INFO_LEN])
                if proc_rows:
                    pa = dict(zip(_PROC_FIELDS, v[_INFO_LEN:_INFO_LEN + plen]))
                    for f in _PROC_INT_FIELDS:
                        pa[f] = int(round(pa[f]))
                    proc_aggs[p * self.L + l] = pa
                srow.extend(v[_INFO_LEN + plen:])
            if spec is not None:
                spec.append(srow)
        ranks = sorted(infos)
        hw.append(_time.perf_counter())
        if ev:
            ev[1].record()

        # If on every rank the time and the memory candidates are the very same rows (the
        # common case: ring not longer than the window, every step has memory), one
        # alignment serves both sections.
        merged = all(d["n_cand"][0] == d["n_cand"][1] == d["n_both"] for d in infos.values())
        t_res = self._align(KIND_TIME, window, infos, ranks, stream, spec=spec)
        if merged:
            m_res = KindResult(observed=t_res.observed, used=list(t_res.used), n_common=t_res.n_common,
                               start_step=t_res.start_step, end_step=t_res.end_step,
                               windows=dict(t_res.windows))
        else:
            m_res = self._align(KIND_MEM, window, infos, ranks, stream)
        hw.append(_time.perf_counter())
        if ev:
            ev[2].record()

        # ---- stage 4: exchange + per-step reduce
        same = (t_res.n_common > 0 and t_res.n_common == m_res.n_common
                and t_res.start_step == m_res.start_step and t_res.end_step == m_res.end_step
                and t_res.used == m_res.used)
        mode = self._exchange_mode(t_res.n_common or m_res.n_common)
        if same:
            self._reduce_pass(KIND_TIME, _abi.MASK_TIME | _abi.MASK_MEM, t_res, stream, mode)
            m_res.series, m_res.shard = t_res.series, t_res.shard
        else:
            if t_res.n_common:
                self._reduce_pass(KIND_TIME, _abi.MASK_TIME, t_res, stream,
                                  self._exchange_mode(t_res.n_common))
            if m_res.n_common:
                self._reduce_pass(KIND_MEM, _abi.MASK_MEM, m_res, stream,
                                  self._exchange_mode(m_res.n_common))
        if mode == "p2p":
            self._p2p_warm = True
        if overlap is not None:  # the GPU is busy with K4: free host time
            overlap(proc_aggs)
        hw.append(_time.perf_counter())
        if ev:
            ev[3].record()

        # ---- stage 5: trend bands
        self._bands(t_res, m_res, same, stream)
        hw.append(_time.perf_counter())
        for i, nm in enumerate(("prepare", "align", "reduce", "bands")):
            timings["host_" + nm] = (hw[i + 1] - hw[i]) * 1e3
        if ev:
            ev[4].record()
            torch.cuda.synchronize(dev)
            names = ["prepare", "align", "reduce", "bands"]
            for i, nm in enumerate(names):
                timings[nm] = float(ev[i].elapsed_time(ev[i + 1]))
            timings["total"] = float(ev[0].elapsed_time(ev[4]))
            timings["k3a_stage"] = float(k3a_ev0.elapsed_time(k3a_ev))
            timings["k3a"] = max((d.get("kernel_ms", 0.0) for d in local_infos), default=0.0) \
                or timings["k3a_stage"]
            timings["k4"] = float(sum(a.elapsed_time(b) for a, b in self._k4_events))
        elif dev.type == "cuda":  # the bands stage synchronised: both kernels have finished
            timings["k3a"] = max((d.get("kernel_ms", 0.0) for d in local_infos), default=0.0)
            if t_res.n_common or m_res.n_common:
                timings["k4"] = float(sum(max(0.0, e.kernel_ms(1)) for e in self.engines
                                          if hasattr(e, "kernel_ms")))
        return ReduceOutput(window=window, ranks=ranks, infos=infos, time=t_res, mem=m_res,
                            exchange=mode, fused_pass=same, timings_ms=timings, proc_aggs=proc_aggs)

    # ------------------------------------------------------------------ memory candidate limit
    def _limit_memory_candidates(self, engine, info: Dict[str, Any], window: int, stream) -> None:
        """Only the newest ``max(20 W, W + 1)`` distinct step ids of a rank enter the memory
        alignment (step_memory/loader.py:215, oracle candidate_rows).  The ring normally holds
        1.5 W rows, so this binds only for a small window over a long ring; then the rank
        advertises the step id of its limit-th newest candidate as its lower bound -- every
        later stage works on [max lo, min hi] and never sees the older candidates."""
        limit = max(20 * window, window + 1)
        if info["n_cand"][KIND_MEM] <= limit:
            return
        lo, hi = info["lo"][KIND_MEM], info["hi"][KIND_MEM]
        if info["dense"][KIND_MEM]:  # consecutive ids
            thr = hi - limit + 1
        else:                        # holes / re-flushed ids: select the newest `limit` of its own
            span = hi - lo + 1
            own = torch.empty(span, dtype=torch.uint8, device=self.device)
            engine.win_presence(KIND_MEM, lo, span, own, stream)
            thr = int(engine.win_select(KIND_MEM, lo, span, own, limit, stream).start_step)
        info["lo"][KIND_MEM] = int(thr)
        info["n_cand"][KIND_MEM] = int(limit)

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

    def run_native(self, window: int, proc_rows: Optional[int], stream: Optional[int] = None):
        """tml_reduce_run on this process's engine; the raw result struct (valid until the next run)."""
        eng = self.engines[0]
        world = self.comm.world
        ptr = self.comm.nccl_comm_ptr(self.device) if world > 1 else 0
        xchg = self.exchange if self.exchange in _abi.XCHG else "auto"
        if xchg == "auto" and world > 1 and not self._peers_on_this_host():
            xchg = "a2a"  # the native driver's own "auto" assumes one host (p2p from 10^6 rows)
        return eng.reduce_run(window, int(proc_rows or 0), xchg,
                              self.speculate, ptr or 0, self.comm.index, world,
                              _stream_of(self.device) if stream is None else stream)

    def _reduce_native(self, window: int, proc_rows: Optional[int], stream: int) -> ReduceOutput:
        return self.convert_native(self.run_native(window, proc_rows, stream), window, proc_rows)

    @staticmethod
    def native_timings(o) -> Dict[str, float]:
        names = ("prepare", "align", "reduce", "bands", "total")
        t = {"host_" + nm: float(o.stage_ms[i]) for i, nm in enumerate(names)}
        t.update({nm: float(o.stage_ms[i]) for i, nm in enumerate(names)})  # stages end in a sync
        t["k3a"], t["k4"] = float(o.k3a_ms), max(0.0, float(o.k4_ms))
        return t

    def convert_native(self, o, window: int, proc_rows: Optional[int]) -> ReduceOutput:
        R = int(o.n_ranks)
        infos = {r: self._info_dict(o.infos[r]) for r in range(R)}
        proc_aggs: Dict[int, Dict[str, Any]] = {}
        if proc_rows:
            for r in range(R):
                pa = {f: getattr(o.procs[r], f) for f in _PROC_FIELDS}
                for f in _PROC_INT_FIELDS:
                    pa[f] = int(pa[f])
                proc_aggs[r] = pa

        def kind(k) -> KindResult:
            res = KindResult(observed=int(k.observed), n_common=int(k.n_common))
            for i in range(int(k.n_used)):
                r = int(k.used[i])
                res.windows[r] = RankWindow(rank=r, n_rows=int(k.n_rows[i]), t_sums=k.t_sums[i][:],
                                            m_sums=k.m_sums[i][:], info=infos[r])
            res.used = sorted(res.windows)
            if res.windows:
                res.start_step, res.end_step = int(k.start_step), int(k.end_step)
            n = int(k.n_common)
            if k.has_bands:
                res.band_sum = [k.band_sum[s][:] for s in range(16)]
                res.band_cnt = [k.band_cnt[s][:] for s in range(16)]
                res.tail_first, res.tail_last = k.tail_first[:], k.tail_last[:]
                res._lay = (trend_layout(n, min_points=200, warmup_frac=0.10),
                            trend_layout(n, min_points=50, warmup_frac=0.0))
            if k.series and n:
                from .engine import _DevView
                res.series = torch.as_tensor(_DevView(int(k.series), _abi.TML_SERIES_PER_STEP * n),
                                             device=self.device).view(_abi.TML_SERIES_PER_STEP, n)
            res.shard = (int(k.shard_lo), int(k.shard_hi))
            return res

        timings = self.native_timings(o)
        self.last_exchanges = int(o.n_exchanges)
        return ReduceOutput(window=window, ranks=list(range(R)), infos=infos, time=kind(o.time), mem=kind(o.mem),
                            exchange=_abi.XCHG_NAME[int(o.exchange_used)], fused_pass=bool(o.fused_pass),
                            timings_ms=timings, proc_aggs=proc_aggs)

    # ------------------------------------------------------------------ alignment
    def _spec_len(self) -> int:
        """Length of the speculative alignment block in the first exchange (0 = off)."""
        if not self.speculate:
            return 0
        handles = self.comm.world > 1 and self.device.type == "cuda" and (
            self.exchange == "p2p" or (self.exchange == "auto" and self._peers_on_this_host()))
        return _ALIGN_LEN if handles else 15

    def _align(self, kind: int, window: int, infos, ranks, stream, spec=None) -> KindResult:
        res = KindResult()
        part = [r for r in ranks if infos[r]["n_cand"][kind] > 0]
        res.observed = len(part)
        if not part:
            return res
        glo = max(infos[r]["lo"][kind] for r in part)
        ghi = min(infos[r]["hi"][kind] for r in part)
        if ghi < glo:
            return res
        span = ghi - glo + 1
        dev = self.device
        if all(infos[r]["dense"][kind] for r in part):
            if (spec is not None and span <= window
                    and all(infos[r]["lo"][kind] == glo and infos[r]["hi"][kind] == ghi for r in part)):
                # every participant speculated on exactly [glo, ghi]: its block is the alignment
                return self._parse_aligns(res, spec, self._spec_len(), part, infos)
            # lock-step fast path: every participant holds every step id of [glo, ghi]
            n_common = min(span, window)
            first = ghi - n_common + 1
            flat: List[float] = []
            for l, e in enumerate(self.engines):
                a = e.win_select_dense(kind, first, n_common, stream)
                flat.extend(self._align_pack(e, kind, a))
            return self._collect_aligns(kind, res, flat, part, infos)
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
        return self._collect_aligns(kind, res, flat, part, infos)

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

    def _collect_aligns(self, kind, res, flat, part, infos) -> KindResult:
        # n_common is identical on every rank, so every rank packed the same layout
        alen = _ALIGN_LEN if len(flat) == _ALIGN_LEN * self.L else 15
        return self._parse_aligns(res, self.comm.all_gather_vec(flat, self.device), alen, part, infos)

    def _parse_aligns(self, res, rows, alen, part, infos) -> KindResult:
        res.handles = {}
        gathered = []
        p2p = alen == _ALIGN_LEN
        for row in rows:
            lst = []
            for l in range(self.L):
                v = row[l * alen:(l + 1) * alen]
                lst.append({"n_common": int(round(v[0])), "start": int(round(v[1])),
                            "end": int(round(v[2])), "n_rows": int(round(v[3])),
                            "t_sums": list(v[4:11]), "m_sums": list(v[11:15]),
                            "handle": bytes(int(round(b)) for b in v[15:87]) if p2p else b""})
            gathered.append(lst)
        n_common = max(a["n_common"] for lst in gathered for a in lst)
        res.n_common = n_common
        if n_common == 0:
            return res
        for p, lst in enumerate(gathered):
            for l, a in enumerate(lst):
                r = p * self.L + l
                if r in part and a["n_rows"] > 0:
                    res.windows[r] = RankWindow(rank=r, n_rows=a["n_rows"], t_sums=a["t_sums"],
                                                m_sums=a["m_sums"], info=infos[r])
                    res.handles[r] = a["handle"]
                    res.start_step, res.end_step = a["start"], a["end"]
        res.used = sorted(res.windows)
        return res

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

    def _reduce_pass(self, kind: int, mask: int, res: KindResult, stream, mode: str) -> None:
        n = res.n_common
        used = res.used
        R = len(used)
        dev = self.device
        # series buffer of this process: [16, n]; only this process's shard is written
        series = torch.empty(_abi.TML_SERIES_PER_STEP * n, dtype=torch.float64, device=dev)
        my = [self._grank(l) for l in range(self.L)]
        # rows handle per used rank
        rows: Dict[int, Any] = {}
        local_used = [r for r in used if r in my]
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
                    rows[r] = e0.peer_open(res.handles[r])
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
        res.series = series.view(_abi.TML_SERIES_PER_STEP, n)
        res.shard = (lo_first or 0, hi_last or 0)

    # ------------------------------------------------------------------ bands
    def _bands(self, t_res: KindResult, m_res: KindResult, same: bool, stream) -> None:
        def run(res: KindResult, kinds):
            n = res.n_common
            if n == 0 or res.series is None:
                return
            a = _abi.BandArgs()
            a.n_common = n
            a.shard_lo, a.shard_hi = res.shard
            lay_t = trend_layout(n, min_points=200, warmup_frac=0.10)
            lay_m = trend_layout(n, min_points=50, warmup_frac=0.0)
            for k, lay in ((0, lay_t), (1, lay_m)):
                for b in range(3):
                    a.band_lo[k][b] = lay[b][0] if lay else 0
                    a.band_hi[k][b] = lay[b][1] if lay else 0
            a.tail_first[0] = 0
            a.tail_first[1] = n - min(n, 1000)
            out = self.engines[0].win_bands(res.series, a, stream)
            vec = ([float(out.sum[s][b]) for s in range(16) for b in range(3)]
                   + [float(out.cnt[s][b]) for s in range(16) for b in range(3)]
                   + [float(out.tail_first[s]) for s in range(16)]
                   + [float(out.tail_last[s]) for s in range(16)])
            parts = []
            for row in self.comm.all_gather_vec(vec, self.device):
                parts.append({
                    "sum": [[row[s * 3 + b] for b in range(3)] for s in range(16)],
                    "cnt": [[int(round(row[48 + s * 3 + b])) for b in range(3)] for s in range(16)],
                    "tf": row[96:112], "tl": row[112:128]})
            res.band_sum = [[sum(p["sum"][s][b] for p in parts) for b in range(3)] for s in range(16)]
            res.band_cnt = [[sum(p["cnt"][s][b] for p in parts) for b in range(3)] for s in range(16)]

            def pick(key, s):
                for p in parts:
                    v = p[key][s]
                    if not math.isnan(v):
                        return v
                return float("nan")

            res.tail_first = [pick("tf", s) for s in range(16)]
            res.tail_last = [pick("tl", s) for s in range(16)]
            res._lay = (lay_t, lay_m)

        run(t_res, (0,))
        if same:
            m_res.band_sum, m_res.band_cnt = t_res.band_sum, t_res.band_cnt
            m_res.tail_first, m_res.tail_last = t_res.tail_first, t_res.tail_last
            m_res._lay = getattr(t_res, "_lay", (None, None))
        else:
            run(m_res, (1,))


__all__ = ["WindowReducer", "LocalComm", "TorchDistComm", "ReduceOutput", "KindResult",
           "RankWindow", "trend_layout"]
