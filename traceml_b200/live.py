"""Live tick: the GPU twin of the reference's ``StepCombinedComputer``.

The reference's live CLI / dashboard recompute, every render tick, the combined
step-time view from SQLite (``src/traceml/renderers/step_time/compute.py:38-315``):
load the last ``4 x window`` rows per rank, intersect the step ids, sum each phase
over the last ``window`` common steps per rank, and build median / worst / sum series.
Here every rank's rows never leave its HBM ring: the tick is four small kernels per
rank on a side stream (``csrc/tml_combined.cuh``), one MIN all-reduce of the presence
bytes, two small vector all-gathers and one row all-gather over NVLink.  Nothing
touches the training stream.

Same class name, constructor meaning, ``compute_cli`` / ``compute_dashboard`` entry
points, stale handling and result shape (``asdict(StepCombinedTimeResult)``) as the
reference; only the data source differs (engines + a comm instead of a db path).

``StepMemoryMetricsComputer`` is the same for the step-memory panel
(``renderers/step_memory/{computer,cli_compute,common}.py``).
"""

from __future__ import annotations

import time
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _abi
from .reduce import LocalComm

KIND_TIME, KIND_MEM = _abi.KIND_TIME, _abi.KIND_MEM

# renderers/step_time/schema.py / compute.py:25-36 -- phase order of the 64-B row
DEFAULT_METRIC_KEYS = ("dataloader_fetch", "h2d", "forward", "backward", "optimizer_step", "step_time")
DEFAULT_HEATMAP_KEYS = ("dataloader_fetch", "h2d", "forward", "backward", "optimizer_step",
                        "wait_proxy", "step_time")
_COL = {k: i for i, k in enumerate(DEFAULT_METRIC_KEYS)}
_INFO_LEN = 7
_ALIGN_LEN = 10


def _empty(msg: str) -> Dict[str, Any]:
    return {"metrics": [], "status_message": msg, "rank_heatmap": None}


class _TickStages:
    """The device stages both live views share (``csrc/tml_combined.cuh``): bounds
    exchange, presence intersection, select + per-rank window values, row exchange and
    the per-step series kernel.  ``self.engines / comm / L / device`` come from the user."""

    def _sid(self) -> int:
        if self.device.type != "cuda":
            return 0
        return int(torch.cuda.current_stream(self.device).cuda_stream)

    def _bounds(self, kind: int, lookback: int, sid: int) -> Dict[int, List[int]]:
        """K7a per local rank + one small all-gather:
        rank -> [n_rows, n_cand, lo, hi, latest, first_step, truncated]."""
        flat: List[float] = []
        for e in self.engines:
            i = e.combined_prepare(kind, lookback, sid)
            flat += [int(i.n_rows), int(i.n_cand), int(i.lo), int(i.hi), int(i.latest_step),
                     int(i.first_step), int(i.truncated)]
        infos: Dict[int, List[int]] = {}
        for p, row in enumerate(self.comm.all_gather_vec(flat, self.device)):
            for l in range(self.L):
                infos[p * self.L + l] = [int(round(x)) for x in row[l * _INFO_LEN:(l + 1) * _INFO_LEN]]
        return infos

    def _intersect(self, kind: int, glo: int, span: int, window: int, sid: int):
        """K7b presence -> MIN all-reduce -> K7c select.  Returns (n_common, presence,
        local aligns, {rank: [sums x 6, peaks x 2]} for the ranks that own rows)."""
        dev = self.device
        presence = None
        for e in self.engines:
            p = torch.empty(span, dtype=torch.uint8, device=dev)
            e.combined_presence(kind, glo, span, p, sid)
            presence = p if presence is None else torch.minimum(presence, p)
        self.comm.all_reduce_min_(presence)
        flat: List[float] = []
        aligns = []
        for e in self.engines:
            a = e.combined_select(kind, glo, span, presence, window, sid)
            aligns.append(a)
            flat += [int(a.n_common), int(a.n_rows)] + [float(x) for x in a.sums] + [float(x) for x in a.peaks]
        vals: Dict[int, List[float]] = {}
        for p, row in enumerate(self.comm.all_gather_vec(flat, dev)):
            for l in range(self.L):
                v = row[l * _ALIGN_LEN:(l + 1) * _ALIGN_LEN]
                if int(round(v[1])) > 0:
                    vals[p * self.L + l] = [float(x) for x in v[2:10]]
        return int(aligns[0].n_common), presence, aligns, vals

    def _series(self, kind, present, aligns, n, glo, presence, first_col, n_cols, sid):
        """One row exchange (all-gather of n x 64 B per rank), then every rank reduces the
        small window itself: [n_cols][median, worst, sum][n] + the step ids."""
        dev = self.device
        local = torch.zeros(self.L, n * 8, dtype=torch.float64, device=dev)
        owner = None
        for l, e in enumerate(self.engines):
            if int(aligns[l].n_rows) > 0:
                local[l].copy_(e.combined_rows_tensor(kind, n))
                owner = e if owner is None else owner
        if self.comm.world == 1:
            allrows = local.view(1, self.L, n * 8)
        else:
            allrows = torch.empty(self.comm.world, self.L, n * 8, dtype=torch.float64, device=dev)
            self.comm.all_gather_into(allrows.view(-1), local.view(-1))
        ptrs = [allrows[r // self.L, r % self.L].data_ptr() for r in present]
        out = torch.empty(n_cols * 3, n, dtype=torch.float64, device=dev)
        self.engines[0].combined_series(ptrs, n, first_col, n_cols, out, sid)
        series = out.cpu().numpy()
        if owner is not None:
            steps = owner.combined_steps(kind, n, sid)
        else:  # this process holds no rows: the reduced presence bytes name the steps
            steps = (torch.nonzero(presence).flatten()[-n:] + glo).cpu().tolist()
        return series, [int(s) for s in steps]


class StepCombinedComputer(_TickStages):
    """compute.py:38-128 (constructor, ``compute_cli``, ``compute_dashboard``, ``_compute``)."""

    def __init__(self, engines: Sequence[Any], comm: Any = None, *, window_size: int = 100,
                 metric_keys: Optional[Sequence[str]] = None,
                 heatmap_keys: Optional[Sequence[str]] = None,
                 stale_ttl_s: Optional[float] = 30.0, lookback_factor: int = 4,
                 device: Optional[torch.device] = None, use_side_stream: bool = True) -> None:
        self.engines = list(engines)
        self.comm = comm or LocalComm()
        self.L = len(self.engines)
        self.window_size = max(1, int(window_size))
        self.metric_keys = list(metric_keys) if metric_keys is not None else list(DEFAULT_METRIC_KEYS)
        self.heatmap_keys = list(heatmap_keys) if heatmap_keys is not None else list(DEFAULT_HEATMAP_KEYS)
        unknown = [k for k in self.metric_keys if k not in _COL]
        if unknown:
            raise ValueError(f"unknown step-time metric keys: {unknown}")
        self.lookback_factor = max(1, int(lookback_factor))
        self.device = device or torch.device("cuda", self.engines[0].device)
        self._stream = None
        if use_side_stream and self.device.type == "cuda":
            self._stream = torch.cuda.Stream(device=self.device)
        self._last_ok: Optional[Dict[str, Any]] = None
        self._last_ok_ts = 0.0
        self._stale_ttl_s = float(stale_ttl_s) if stale_ttl_s is not None else None
        self.last_timings_ms: Dict[str, float] = {}

    # ------------------------------------------------------------------ public API
    def compute_cli(self) -> Dict[str, Any]:
        return self._compute(include_series=True, include_rank_heatmap=False)

    def compute_dashboard(self) -> Dict[str, Any]:
        return self._compute(include_series=False, include_rank_heatmap=True)

    def _compute(self, *, include_series: bool, include_rank_heatmap: bool) -> Dict[str, Any]:
        """compute.py:103-123.  The tick is a collective: an exception on one rank is
        an exception on all (the native calls fail identically or not at all)."""
        try:
            if self._stream is not None:
                with torch.cuda.stream(self._stream):
                    result = self._compute_impl(include_series=include_series,
                                                include_rank_heatmap=include_rank_heatmap)
            else:
                result = self._compute_impl(include_series=include_series,
                                            include_rank_heatmap=include_rank_heatmap)
        except Exception as exc:  # noqa: BLE001 -- the live view must never take training down
            return self._stale_or_empty(f"STALE (exception: {type(exc).__name__})")
        if not result["metrics"]:
            return self._stale_or_empty("STALE (no metrics this tick)")
        self._last_ok = result
        self._last_ok_ts = time.time()
        return result

    def _stale_or_empty(self, msg: str) -> Dict[str, Any]:
        """compute.py:424-446."""
        if self._last_ok is not None and (self._stale_ttl_s is None
                                          or (time.time() - self._last_ok_ts) <= self._stale_ttl_s):
            return {"metrics": self._last_ok["metrics"], "status_message": msg,
                    "rank_heatmap": self._last_ok["rank_heatmap"]}
        return _empty("No fresh step-combined data")

    # ------------------------------------------------------------------ core
    def _compute_impl(self, *, include_series: bool, include_rank_heatmap: bool) -> Dict[str, Any]:
        t0 = time.perf_counter()
        sid, W = self._sid(), self.window_size
        lookback = max(W * self.lookback_factor, W)  # compute.py:366-368
        infos = self._bounds(KIND_TIME, lookback, sid)
        ranks = sorted(r for r, v in infos.items() if v[0] > 0)  # compute.py:139-143
        if not ranks:
            return _empty("No ranks available")
        completed = min(infos[r][4] for r in ranks)               # compute.py:147
        glo = max(infos[r][2] for r in ranks)
        ghi = min(min(infos[r][3] for r in ranks), completed)
        if ghi < glo:
            return _empty("No common step window yet")
        span = ghi - glo + 1
        n, presence, aligns, vals = self._intersect(KIND_TIME, glo, span, W, sid)
        if n == 0:
            return _empty("No common step window yet")
        sums = {r: v[:6] for r, v in vals.items() if r in ranks}
        present = [r for r in ranks if r in sums]
        coverage = {"expected_steps": W, "steps_used": n, "completed_step": int(completed),
                    "world_size": len(ranks), "ranks_present": len(present),
                    "incomplete": len(present) < len(ranks)}
        steps: List[int] = []
        series = None
        if include_series:  # CLI mode
            series, steps = self._series(KIND_TIME, present, aligns, n, glo, presence, 0, 6, sid)
        result = self._assemble(present, sums, coverage, steps, series, include_rank_heatmap)
        self.last_timings_ms = {"tick": (time.perf_counter() - t0) * 1e3}
        return result

    # ------------------------------------------------------------------ rank-level (O(R) scalars)
    def _assemble(self, present, sums, coverage, steps, series, include_rank_heatmap):
        col = lambda k, r: sums[r][_COL[k]]  # noqa: E731
        by_key: Dict[str, Dict[int, float]] = {k: {r: col(k, r) for r in present}
                                               for k in DEFAULT_METRIC_KEYS}
        # compute.py:177-187
        wait = {r: max(0.0, col("step_time", r) - col("h2d", r) - col("forward", r)
                       - col("backward", r) - col("optimizer_step", r)) for r in present}
        by_key["wait_proxy"] = wait
        # compute.py:189-201
        scores = {r: col("dataloader_fetch", r)
                  + max(col("step_time", r),
                        col("h2d", r) + col("forward", r) + col("backward", r) + col("optimizer_step", r))
                  for r in present}
        worst_rank = max(scores, key=scores.get) if scores else None
        median_rank = None
        if scores:  # compute.py:628-660
            target = float(np.median(np.array(list(scores.values()), dtype=np.float64)))
            median_rank = min(scores, key=lambda r: (abs(scores[r] - target), scores[r], r))

        metrics: Dict[str, Any] = {}
        for k in self.metric_keys:
            ser = None
            if series is not None:
                c = _COL[k]
                ser = {"steps": list(steps), "median": series[c * 3].tolist(),
                       "worst": series[c * 3 + 1].tolist(), "sum": series[c * 3 + 2].tolist()}
            m = self._metric(k, by_key[k], present, coverage, ser)
            if k == "step_time" and worst_rank is not None:
                m["summary"]["worst_rank"] = int(worst_rank)  # compute.py:225-232
            metrics[k] = m
        metrics["wait_proxy"] = self._metric("wait_proxy", wait, present, coverage, None)

        heat = None
        if include_rank_heatmap and metrics:  # compute.py:263-297
            keys = [k for k in self.heatmap_keys if k in by_key]
            rows = [{"rank": int(r), "sums_ms": {k: float(by_key[k].get(r, 0.0)) for k in keys}}
                    for r in present]
            rows.sort(key=lambda row: (scores.get(row["rank"], 0.0), row["sums_ms"].get("step_time", 0.0),
                                       row["sums_ms"].get("dataloader_fetch", 0.0)), reverse=True)
            heat = {"window_size": self.window_size, "steps_used": coverage["steps_used"],
                    "metric_keys": keys, "rows": rows,
                    "sort_by": ["overall_score", "step_time", "dataloader_fetch"]}
        status = "OK"
        if worst_rank is not None:
            status += f" | overall_worst_rank=r{worst_rank}"
        if median_rank is not None:
            status += f" | overall_median_rank=r{median_rank}"
        return {"metrics": list(metrics.values()), "status_message": status, "rank_heatmap": heat}

    @staticmethod
    def _metric(key, rank_sums, ranks, coverage, series):
        """compute.py:533-626."""
        arr = np.array([float(rank_sums.get(r, 0.0)) for r in ranks], dtype=np.float64)
        median_total = float(np.median(arr))
        wi = int(np.argmax(arr))
        worst_total, worst_rank = float(arr[wi]), int(ranks[wi])
        if coverage["ranks_present"] <= 1:
            median_total, skew_ratio, skew_pct = worst_total, 0.0, 0.0
        elif median_total > 0.0:
            skew_ratio = worst_total / median_total
            skew_pct = (worst_total - median_total) / median_total
        else:
            skew_ratio = skew_pct = 0.0
        return {"metric": str(key), "clock": "mixed", "series": series,
                "summary": {"window_size": int(coverage["expected_steps"]),
                            "steps_used": int(coverage["steps_used"]),
                            "median_total": median_total, "worst_total": worst_total,
                            "worst_rank": worst_rank, "skew_ratio": float(skew_ratio),
                            "skew_pct": float(skew_pct)},
                "coverage": coverage}


# =============================================================================== step memory
_MEM_COL = {"peak_allocated": 0, "peak_reserved": 1}
_NO_GPU = "No GPU detected. Step memory uses torch-based GPU memory telemetry."


class StepMemoryCombinedComputer(_TickStages):
    """One window size of the step-memory panel: ``build_step_memory_combined_result``
    (common.py:215-356) + the stale wrapper of ``StepMemoryCLIComputer.compute``
    (cli_compute.py:44-88)."""

    def __init__(self, engines: Sequence[Any], comm: Any = None, *, window_size: int = 100,
                 stale_ttl_s: Optional[float] = 30.0, metric_keys: Sequence[str] = ("peak_allocated",
                                                                                     "peak_reserved"),
                 gpu_available: Optional[bool] = None, device: Optional[torch.device] = None,
                 use_side_stream: bool = True) -> None:
        self.engines = list(engines)
        self.comm = comm or LocalComm()
        self.L = len(self.engines)
        self.window_size = int(window_size)
        self.metric_keys = [k for k in metric_keys]
        self.device = device or torch.device("cuda", self.engines[0].device)
        # the reference reads MAX(gpu_available) from process/system samples (common.py:78-112)
        self.gpu_available = (torch.cuda.is_available() if gpu_available is None and self.device.type == "cuda"
                              else gpu_available)
        self._stream = None
        if use_side_stream and self.device.type == "cuda":
            self._stream = torch.cuda.Stream(device=self.device)
        self._last_ok: Optional[Dict[str, Any]] = None
        self._last_ok_ts = 0.0
        self._stale_ttl_s = float(stale_ttl_s) if stale_ttl_s is not None else None

    def compute(self) -> Dict[str, Any]:
        try:
            if self._stream is not None:
                with torch.cuda.stream(self._stream):
                    out = self._compute_impl()
            else:
                out = self._compute_impl()
        except Exception:  # noqa: BLE001
            return self._stale_or_empty("STALE (exception)")
        if not out["metrics"]:
            if "No GPU detected" in str(out["status_message"]):  # cli_compute.py:60-64
                self._last_ok, self._last_ok_ts = None, 0.0
                return out
            return self._stale_or_empty("STALE (no metrics this tick)")
        self._last_ok, self._last_ok_ts = out, time.time()
        return out

    def _stale_or_empty(self, msg: str) -> Dict[str, Any]:
        if self._last_ok is not None and (self._stale_ttl_s is None
                                          or (time.time() - self._last_ok_ts) <= self._stale_ttl_s):
            return {"metrics": self._last_ok["metrics"], "status_message": msg}
        return {"metrics": [], "status_message": "No complete memory metrics available"}

    def _compute_impl(self) -> Dict[str, Any]:
        sid = self._sid()
        ws = max(1, int(self.window_size))
        scan_span = max(ws * 20, ws + 1)                     # common.py:245
        lookback = scan_span + 64                            # room for re-flushed step ids
        infos = self._bounds(KIND_MEM, lookback, sid)
        ranks = sorted(r for r, v in infos.items() if v[0] > 0)
        if not ranks:                                        # common.py:235-239
            return {"metrics": [], "status_message": "Waiting for first fully completed step across all ranks…"}
        world_size = len(ranks)
        completed = min(infos[r][4] for r in ranks)
        start = max(0, completed - scan_span + 1)
        # a rank far ahead (or full of re-flushed ids) may need older rows than the first
        # look-back held: widen locally -- its bounds in `infos` do not change
        for l, e in enumerate(self.engines):
            v = infos[self.comm.index * self.L + l]
            lb, first, trunc = lookback, v[5], v[6]
            while trunc and first > start:
                lb *= 4
                i = e.combined_prepare(KIND_MEM, lb, sid)
                first, trunc = int(i.first_step), int(i.truncated)
                if int(i.n_rows) < lb:  # clamped by the ring: nothing older is retained
                    break
        span = completed - start + 1
        n, presence, aligns, vals = self._intersect(KIND_MEM, start, span, ws, sid)
        present = sorted(r for r in vals if r in ranks)
        out: List[Dict[str, Any]] = []
        if n > 0 and present:
            series, steps = self._series(KIND_MEM, present, aligns, n, start, presence, 6, 2, sid)
            for key in self.metric_keys:
                c = _MEM_COL.get(key)
                if c is None:
                    continue
                peaks = np.array([vals[r][6 + c] for r in present], dtype=np.float64)  # common.py:289-300
                median_peak = float(np.median(peaks))
                worst_peak = float(np.max(peaks))
                worst_rank = int(present[int(np.argmax(peaks))])
                skew_ratio = (worst_peak / median_peak) if median_peak > 0.0 else 0.0
                skew_pct = ((worst_peak - median_peak) / median_peak) if median_peak > 0.0 else 0.0
                out.append({
                    "metric": str(key), "device": self._device_label(),
                    "series": {"steps": list(steps), "median": series[c * 3].tolist(),
                               "worst": series[c * 3 + 1].tolist()},
                    "summary": {"window_size": ws, "steps_used": n, "median_peak": median_peak,
                                "worst_peak": worst_peak, "worst_rank": worst_rank,
                                "skew_ratio": float(skew_ratio), "skew_pct": float(skew_pct)},
                    "coverage": {"expected_steps": ws, "steps_used": n, "completed_step": int(completed),
                                 "world_size": int(world_size), "ranks_present": len(present),
                                 "incomplete": len(present) < world_size},
                })
        if out:
            status = "OK"
        elif self.gpu_available is False:  # the rank that fixes `completed` has a row in the window
            status = _NO_GPU
        else:
            status = "No complete memory metrics available"
        return {"metrics": out, "status_message": status}

    def _device_label(self) -> Optional[str]:
        """The reference reports the majority device string over ranks, ties broken by
        Python set order (common.py:400-408); one label here only when it is unambiguous."""
        if self.comm.world * self.L == 1 and self.device.type == "cuda":
            return f"cuda:{self.device.index or 0}"
        return None


class StepMemoryMetricsComputer:
    """computer.py:20-50: the facade the renderers hold."""

    def __init__(self, engines: Sequence[Any], comm: Any = None, *, stale_ttl_s: Optional[float] = 30.0,
                 cli_window_size: int = 400, dashboard_window_size: int = 400, **kw: Any) -> None:
        self._cli = StepMemoryCombinedComputer(engines, comm, window_size=cli_window_size,
                                               stale_ttl_s=stale_ttl_s, **kw)
        self._dashboard = StepMemoryCombinedComputer(engines, comm, window_size=dashboard_window_size,
                                                     stale_ttl_s=stale_ttl_s, **kw)

    def compute_cli(self) -> Dict[str, Any]:
        return self._cli.compute()

    def compute_dashboard(self) -> Dict[str, Any]:
        return self._dashboard.compute()
