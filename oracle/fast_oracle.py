"""Oracle for LARGE windows: the load / align / per-step-reduce stages of the
Step-Time and Step-Memory sections restated with numpy.  TEST INFRASTRUCTURE ONLY
(tests/, __graft_entry__.smoke(), bench.py's parity + cpu_baseline legs).

The row-level restatement (``step_time_oracle.py`` / ``step_memory_oracle.py``) walks every row
in Python: fine up to ~2*10^5 rows, hopeless at bench.py's W = 4*10^6.  This module
vectorises exactly the O(R*W) stages and then hands over to the SAME downstream functions
(``step_time_oracle.diagnose_summary / global_points / overview``,
``step_memory_oracle.diagnose_summary / rollup_points``), so labels, rank ids and strings come
from the pinned code.  It is itself pinned: ``tests/test_fast_oracle_cpu.py`` requires bit
equality (``==`` on floats) with the row-level oracle on every step golden case plus seeded
random windows, which in turn is pinned ``==`` against the unmodified reference
(``tests/golden/make_golden.py``).

What keeps it bit-exact with the reference (file:line = the reference's src/traceml/...):
  * ns -> ms is IEEE division ``ns / 1e6`` (the wire rows carry ``duration_ms`` computed that way);
  * per-rank window sums are the reference's plain ``s += x`` loops over rows in DESCENDING step
    order (reporting/sections/step_time/model.py:241-268, loader.py ``ORDER BY step DESC``;
    alignment.py:59-75 iterates the same dict order): ``np.add.accumulate`` is a strictly
    sequential IEEE sum, unlike ``np.sum`` (pairwise);
  * step-memory rank means are ``sum(...) / len(...)`` over Python floats
    (reporting/sections/step_memory/model.py:224-246): CPython >= 3.12 ``sum`` is
    Neumaier-compensated, i.e. the correctly rounded exact sum for integer-valued byte counts --
    computed here as an exact Python-int sum converted once;
  * per-step cross-rank median / max: ``np.median`` / ``np.max`` over the rank axis
    (diagnostics/step_time/adapters.py:92-139); memory median = mean of the two middles
    (step_memory/model.py:130-138), which is what ``np.median`` computes too.

Scope: every rank's candidate rows have unique step ids (no re-flushed failed steps); holes and
ragged ranks are fine.  Duplicated step ids -> ``NotImplementedError`` (use the row-level oracle).
The trend / creep rules read only the last 10 000 points of a series
(analytics/trends/core.py:51-84 ``history_limit``), so the series handed downstream are the
last ``min(n, 10 000)`` aligned steps; ``series_at`` gives any other steps for point checks.
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import numpy as np

from . import step_memory_oracle as smo
from . import step_time_oracle as sto

TAIL = 10_000  # history_limit of the trend evidence (analytics/trends/core.py:58)
FLAG_HAS_MEM = 1

# WindowRow columns (SURVEY 8d): dl, h2d, fwd, bwd, opt, wall (ms), peak_alloc, peak_resv (B)
C_DL, C_H2D, C_FWD, C_BWD, C_OPT, C_WALL, C_ALLOC, C_RESV = range(8)


def seq_sum(x: np.ndarray) -> float:
    """One IEEE add after another, in array order, starting from 0.0."""
    if x.size == 0:
        return 0.0
    return float(np.add.accumulate(x, dtype=np.float64)[-1])


def window_rows(records: np.ndarray) -> np.ndarray:
    """StepRecords -> [n, 8] f64 WindowRows (what K3a produces)."""
    out = np.empty((len(records), 8), dtype=np.float64)
    out[:, :6] = records["dur_ns"].astype(np.float64) / 1.0e6
    out[:, 6] = records["peak_alloc"].astype(np.float64)
    out[:, 7] = records["peak_resv"].astype(np.float64)
    return out


def derived(rows: np.ndarray) -> Dict[str, np.ndarray]:
    """model.py:241-256 per row, same expression order."""
    dl, f, b, o, cpu = rows[:, C_DL], rows[:, C_FWD], rows[:, C_BWD], rows[:, C_OPT], rows[:, C_WALL]
    compute = (f + b) + o
    traced = np.maximum(cpu, compute)
    wait = np.maximum(0.0, traced - compute)
    return {"dataloader_fetch": dl, "forward": f, "backward": b, "optimizer_step": o,
            "step_time": traced, "wait_proxy": wait, "_cpu": cpu, "_compute": compute}


def _check_unique(steps: np.ndarray) -> None:
    if steps.size > 1 and np.any(steps[1:] == steps[:-1]):
        raise NotImplementedError("duplicated step ids: use the row-level oracle")
    if steps.size > 1 and np.any(steps[1:] < steps[:-1]):
        raise ValueError("step ids decrease")


def rank_part(records: np.ndarray, max_rows: int) -> Optional[Dict[str, Any]]:
    """One rank's share of ``load_section``: the last ``max_rows`` rows (loader.py:44-72), the
    usable ones (model.py:188-196), their reference-order sums (model.py:262-281)."""
    if len(records) == 0:
        return None
    recs = records[-max(1, int(max_rows)):]
    steps = recs["step"].astype(np.int64)
    _check_unique(steps)
    rows = window_rows(recs)
    d = derived(rows)
    usable = (d["dataloader_fetch"] > 0) | (d["forward"] > 0) | (d["backward"] > 0) | \
             (d["optimizer_step"] > 0) | (d["_cpu"] > 0)
    if not usable.any():
        return None
    idx = np.nonzero(usable)[0][::-1]  # newest first
    n = int(idx.size)
    sums = [seq_sum(d[k][idx]) for k in ("dataloader_fetch", "forward", "backward", "optimizer_step", "_cpu", "step_time")]
    sums.append(seq_sum((d["dataloader_fetch"] + d["step_time"])[idx]))
    return {"n": n, "sums": sums, "steps": steps[usable], "rows": rows[usable],
            "summary": sto._summary(n, *sums)}


def aligned_part(part: Dict[str, Any], common: np.ndarray) -> Dict[str, Any]:
    """alignment.py:44-91 for one rank over the common steps (newest first)."""
    pos = np.searchsorted(part["steps"], common)
    rows = part["rows"][pos]
    d = derived(rows)
    order = slice(None, None, -1)
    st = d["step_time"]
    compute = d["_compute"]
    traced = np.maximum(st, compute)
    sums = [seq_sum(d["dataloader_fetch"][order]), seq_sum(d["forward"][order]), seq_sum(d["backward"][order]),
            seq_sum(d["optimizer_step"][order]), seq_sum(np.maximum(0.0, st)[order]), seq_sum(traced[order]),
            seq_sum((d["dataloader_fetch"] + traced)[order])]
    return {"rows": rows, "sums": sums, "summary": sto._summary(int(common.size), *sums)}


def common_suffix(step_sets: Sequence[np.ndarray], max_rows: int) -> np.ndarray:
    """utils/step_windows.py:14-33."""
    if not step_sets or any(s.size == 0 for s in step_sets):
        return np.zeros(0, dtype=np.int64)
    common = step_sets[0]
    for s in step_sets[1:]:
        common = np.intersect1d(common, s, assume_unique=True)
    return common[-max(1, int(max_rows)):]


def series16(rows_by_rank: np.ndarray) -> np.ndarray:
    """[R, k, 8] aligned rows -> [16, k]: metric m -> (2m: median, 2m+1: worst); metric order
    dataloader, forward, backward, optimizer, step(traced), wait, alloc, resv (K4's layout)."""
    R, k, _ = rows_by_rank.shape
    out = np.empty((16, k), dtype=np.float64)
    f, b, o = rows_by_rank[:, :, C_FWD], rows_by_rank[:, :, C_BWD], rows_by_rank[:, :, C_OPT]
    compute = (f + b) + o
    traced = np.maximum(rows_by_rank[:, :, C_WALL], compute)
    wait = np.maximum(0.0, traced - compute)
    cols = [rows_by_rank[:, :, C_DL], f, b, o, traced, wait, rows_by_rank[:, :, C_ALLOC], rows_by_rank[:, :, C_RESV]]
    for m, v in enumerate(cols):
        out[2 * m] = np.median(v, axis=0)
        out[2 * m + 1] = np.max(v, axis=0)
    return out


_TIME_KEYS = ("dataloader_fetch", "forward", "backward", "optimizer_step", "step_time", "wait_proxy")


def step_time_from_parts(parts: Dict[int, Optional[Dict[str, Any]]], aligned: Dict[int, Dict[str, Any]],
                         common_n: int, start: Optional[int], end: Optional[int], max_rows: int,
                         tail_series: Optional[np.ndarray], tail_steps: Optional[np.ndarray],
                         latest_step: Optional[int]) -> Dict[str, Any]:
    """Everything after the O(R*W) stages, through the pinned row-level oracle's functions."""
    per_rank_summary = {r: p["summary"] for r, p in sorted(parts.items()) if p is not None}
    observed = len(per_rank_summary)
    a_sum = {r: a["summary"] for r, a in sorted(aligned.items())}
    window = {"alignment": "common_steps", "steps_analyzed": int(common_n if a_sum else 0),
              "start_step": start if a_sum else None, "end_step": end if a_sum else None,
              "window_size": max(1, int(max_rows)), "global_ranks_used": len(a_sum),
              "global_ranks_observed": observed}
    pre = None
    if a_sum and tail_series is not None:
        ser = {}
        for m, key in enumerate(_TIME_KEYS):
            ser[key] = {"steps": [int(s) for s in tail_steps], "median": tail_series[2 * m].tolist(),
                        "worst": tail_series[2 * m + 1].tolist()}
        pre = {"steps_used": int(common_n), "completed_step": int(end), "series": ser}
    diag = sto.diagnose_summary(sto.rank_signals_from_summary(a_sum), max_rows=max(1, int(max_rows)),
                                precomputed=pre) if a_sum else None
    return {"data": {"training_steps": (latest_step + 1) if latest_step is not None else 0,
                     "latest_step_observed": latest_step, "aligned_summary": a_sum,
                     "aligned_window": window, "per_global_rank_summary": per_rank_summary,
                     "max_rows": max(1, int(max_rows))},
            "diagnosis": diag, "global": sto.global_points(a_sum), "overview": sto.overview(a_sum)}


def step_time_section(records_by_rank: Dict[int, np.ndarray], *, max_rows: int = 10_000) -> Dict[str, Any]:
    """``step_time_oracle.step_time_section`` for unique-step windows, vectorised; plus
    ``_series`` ([16, n] time columns 0..11 valid) and ``_steps`` for element-wise checks."""
    parts = {int(r): rank_part(recs, max_rows) for r, recs in sorted(records_by_rank.items())}
    live = {r: p for r, p in parts.items() if p is not None}
    latest = max((int(recs["step"].max()) for recs in records_by_rank.values() if len(recs)), default=None)
    common = common_suffix([p["steps"] for p in live.values()], max_rows) if live else np.zeros(0, np.int64)
    aligned = {r: aligned_part(p, common) for r, p in live.items()} if common.size else {}
    ser = None
    if aligned:
        ser = series16(np.stack([aligned[r]["rows"] for r in sorted(aligned)]))
    tail = min(TAIL, int(common.size))
    out = step_time_from_parts(parts, aligned, int(common.size),
                               int(common[0]) if common.size else None,
                               int(common[-1]) if common.size else None, max_rows,
                               ser[:, -tail:] if ser is not None else None,
                               common[-tail:] if common.size else None, latest)
    out["_series"], out["_steps"] = ser, common
    return out


# ----------------------------------------------------------------------------- step memory
def mem_part(records: np.ndarray, window_size: int) -> Optional[Dict[str, Any]]:
    """step_memory/loader.py:112-205: rows with memory, newest ``max(20 W, W+1)`` step ids."""
    has = (records["flags"] & FLAG_HAS_MEM) != 0
    recs = records[has]
    if len(recs) == 0:
        return None
    limit = max(int(window_size) * 20, int(window_size) + 1)
    recs = recs[-limit:]
    steps = recs["step"].astype(np.int64)
    _check_unique(steps)
    return {"steps": steps, "alloc": recs["peak_alloc"].astype(np.uint64), "resv": recs["peak_resv"].astype(np.uint64)}


def step_memory_section(records_by_rank: Dict[int, np.ndarray], *, window_size: int = 10_000,
                        gpu_total_bytes: Optional[float] = None) -> Dict[str, Any]:
    W = max(1, int(window_size))
    parts = {int(r): mem_part(recs, W) for r, recs in sorted(records_by_rank.items())}
    live = {r: p for r, p in parts.items() if p is not None}
    seen = sum(1 for recs in records_by_rank.values() if len(recs))  # loader.py:98-109: any row at all
    steps_all = [int(recs["step"].max()) for recs in records_by_rank.values() if len(recs)]
    latest = max(steps_all) if steps_all else None
    common = common_suffix([p["steps"] for p in live.values()], W) if live else np.zeros(0, np.int64)
    metrics, means, ser = [], {}, None
    ranks = sorted(live)
    if common.size and ranks:
        n = int(common.size)
        cols = {}
        for r in ranks:
            pos = np.searchsorted(live[r]["steps"], common)
            cols[r] = (live[r]["alloc"][pos], live[r]["resv"][pos])
            means[str(r)] = {  # exact integer sum -> one rounding == CPython 3.12 float sum()
                "peak_allocated_bytes": float(int(cols[r][0].sum(dtype=np.uint64))) / n,
                "peak_reserved_bytes": float(int(cols[r][1].sum(dtype=np.uint64))) / n}
        ser = np.empty((4, n), dtype=np.float64)
        tail = min(TAIL, n)
        for idx, name in enumerate(("peak_allocated", "peak_reserved")):
            by_rank = np.stack([cols[r][idx].astype(np.float64) for r in ranks])
            ser[2 * idx] = np.median(by_rank, axis=0)
            ser[2 * idx + 1] = np.max(by_rank, axis=0)
            peaks = [float(v) for v in by_rank.max(axis=1)]
            med_peak, worst_peak = float(smo.median2(peaks)), float(max(peaks))
            worst_rank = int(ranks[peaks.index(worst_peak)])
            metrics.append({
                "metric": name,
                "series": {"steps": [int(s) for s in common[-tail:]], "median": ser[2 * idx, -tail:].tolist(),
                           "worst": ser[2 * idx + 1, -tail:].tolist()},
                "summary": {"window_size": W, "steps_used": n, "median_peak": med_peak, "worst_peak": worst_peak,
                            "worst_rank": worst_rank,
                            "skew_ratio": float(worst_peak / med_peak if med_peak > 0.0 else 0.0),
                            "skew_pct": float((worst_peak - med_peak) / med_peak if med_peak > 0.0 else 0.0)},
                "coverage": {"expected_steps": W, "steps_used": n, "completed_step": int(common[-1]),
                             "world_size": seen, "ranks_present": len(ranks), "incomplete": len(ranks) < seen}})
    return {"training_steps": latest + 1 if latest is not None else 0, "latest_step_observed": latest,
            "window": {"steps_first": int(common[0]) if common.size else None,
                       "steps_last": int(common[-1]) if common.size else None, "n_steps": int(common.size),
                       "window_size": W, "global_ranks_seen": seen, "global_ranks_used": len(means)},
            "metrics": metrics, "per_global_rank": means,
            "diagnosis": smo.diagnose_summary(metrics, gpu_total_bytes), "global": smo.rollup_points(means),
            "_series": ser, "_steps": common}


__all__ = ["step_time_section", "step_memory_section", "rank_part", "aligned_part", "mem_part", "common_suffix",
           "series16", "window_rows", "seq_sum", "step_time_from_parts"]
