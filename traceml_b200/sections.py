"""Step-Time / Step-Memory / Process sections from the device-side reduce.

The GPU-native counterpart of
``src/traceml/reporting/sections/{step_time,step_memory,process}/__init__.py``
(``load -> to_diagnosis_input -> diagnose``): ``load`` is the cross-rank window
reduce on the GPUs (``reduce.WindowReducer``), ``diagnose`` is the C++ rule
engine (``csrc/tml_diag.cpp``).  The objects returned here are plain dicts with
the reference's field names; ``reporting.py`` turns them into the reference's
own dataclasses for the kept payload builders.  With one engine per process the same
objects come from ``tml_sections_json`` (``csrc/tml_sections.cpp``) in one JSON parse;
this module is then the specification the native emitter is tested against.

Also holds the O(R) public rollups the payload uses
(``reporting/sections/step_time/model.py:77-105,284-498``,
``step_memory/model.py:322-412``).
"""

from __future__ import annotations

import math
import os
import statistics
from typing import Any, Dict, List, Optional, Sequence

from . import _abi
from .reduce import KIND_MEM, KIND_TIME, KindResult, ReduceOutput, WindowReducer, _stream_of

# series index = metric * 2 + {0: median, 1: worst}
S_DL, S_FWD, S_BWD, S_OPT, S_STEP, S_WAIT, S_ALLOC, S_RESV = range(8)


def _summary_from_sums(n: int, s: Sequence[float]) -> Dict[str, Any]:
    """RankStepSummary (reporting/sections/step_time/model.py:108-120,270-281)."""
    return {
        "steps_analyzed": int(n),
        "avg_dataloader_ms": s[0] / n,
        "avg_forward_ms": s[1] / n,
        "avg_backward_ms": s[2] / n,
        "avg_optimizer_ms": s[3] / n,
        "avg_step_cpu_ms": s[4] / n,
        "avg_traced_step_ms": s[5] / n,
        "avg_gpu_compute_ms": ((s[1] + s[2]) + s[3]) / n,
        "avg_total_step_ms": s[6] / n,
    }


def _trend_in(res: KindResult, series: int, kind: int) -> _abi.TrendIn:
    t = _abi.TrendIn()
    lay = getattr(res, "_lay", (None, None))[kind]
    if res.band_sum is None or lay is None:
        t.valid = 0
        return t
    cnt = res.band_cnt[series]
    if min(cnt) <= 0:
        t.valid = 0
        return t
    t.valid = 1
    t.baseline_avg = res.band_sum[series][0] / cnt[0]
    t.mid_avg = res.band_sum[series][1] / cnt[1]
    t.recent_avg = res.band_sum[series][2] / cnt[2]
    return t


# ----------------------------------------------------------------------------- step time
def closest_rank_to_median(values: Dict[int, float]) -> Optional[int]:
    """model.py:77-105 -- tie-break |delta|, value, rank."""
    if not values:
        return None
    med = statistics.median(float(v) for v in values.values())
    return min(values, key=lambda r: (abs(float(values[r]) - med), float(values[r]), r))


def wait_avg_ms(s: Dict[str, Any]) -> float:
    """model.py:284-307."""
    return max(0.0, s["avg_traced_step_ms"]
               - (s["avg_forward_ms"] + s["avg_backward_ms"] + s["avg_optimizer_ms"]))


def step_time_global(summary_by_rank: Dict[int, Dict[str, Any]]) -> Dict[str, Any]:
    """average / median{value,idx} / worst{value,idx} (model.py:310-403)."""
    cols = {
        "total_step_ms": "avg_total_step_ms", "dataloader_ms": "avg_dataloader_ms",
        "compute_ms": "avg_gpu_compute_ms", "wait_ms": None, "forward_ms": "avg_forward_ms",
        "backward_ms": "avg_backward_ms", "optimizer_ms": "avg_optimizer_ms",
    }
    avg, med, worst = {}, {}, {}
    for metric, key in cols.items():
        vals = {int(r): (wait_avg_ms(s) if key is None else float(s[key]))
                for r, s in summary_by_rank.items()}
        if not vals:
            avg[metric] = None
            med[metric] = worst[metric] = {"value": None, "idx": None}
            continue
        vs = list(vals.values())
        avg[metric] = sum(vs) / len(vs)
        mr = closest_rank_to_median(vals)
        wr = max(vals, key=lambda r: (vals[r], -int(r)))
        med[metric] = {"value": vals[mr], "idx": str(mr)}
        worst[metric] = {"value": vals[wr], "idx": str(wr)}
    return {"average": avg, "median": med, "worst": worst}


def step_time_overview(summary_by_rank: Dict[int, Dict[str, Any]]) -> Dict[str, Any]:
    """model.py:445-498."""
    if not summary_by_rank:
        return {"rank_comparison": "no_data", "median_global_rank": None,
                "worst_global_rank": None, "median_avg_step_ms": None,
                "worst_avg_step_ms": None, "step_time_skew_percent": None}
    tot = {r: s["avg_total_step_ms"] for r, s in summary_by_rank.items()}
    wr = max(tot, key=tot.get)
    mr = closest_rank_to_median(tot)
    w, m = tot[wr], tot[mr]
    skew = 100.0 * (w - m) / m if (m > 0.0 and wr != mr) else None
    return {"rank_comparison": "single_rank" if len(tot) <= 1 else "distributed",
            "median_global_rank": mr, "worst_global_rank": wr,
            "median_avg_step_ms": m, "worst_avg_step_ms": w, "step_time_skew_percent": skew}


def build_step_time(out: ReduceOutput) -> Dict[str, Any]:
    res = out.time
    infos = out.infos
    have = [r for r in out.ranks if infos[r]["n_retained"] > 0]
    latest = max((infos[r]["latest_step"] for r in have), default=None)
    per_rank = {r: _summary_from_sums(infos[r]["t_count"], infos[r]["t_sums"])
                for r in out.ranks if infos[r]["t_count"] > 0}
    aligned = {r: _summary_from_sums(w.n_rows, w.t_sums) for r, w in sorted(res.windows.items())}
    window = {
        "alignment": "common_steps", "steps_analyzed": int(res.n_common if aligned else 0),
        "start_step": res.start_step if aligned else None,
        "end_step": res.end_step if aligned else None,
        "window_size": int(out.window), "global_ranks_used": len(aligned),
        "global_ranks_observed": int(res.observed),
    }
    data = {
        "training_steps": (latest + 1) if latest is not None else 0,
        "latest_step_observed": latest,
        "aligned_summary": aligned,
        "aligned_window": window,
        "per_global_rank_summary": per_rank,
        "max_rows": int(out.window),
    }
    # ---- diagnosis (host C++)
    din = _abi.StDiagIn()
    din.n_ranks = len(aligned)
    din.max_rows = int(out.window)
    din.n_common = int(res.n_common if aligned else 0)
    din.completed_step = int(res.end_step or 0)
    for i, (r, s) in enumerate(sorted(aligned.items())):
        rm = din.ranks[i]
        rm.rank, rm.steps_analyzed = int(r), int(s["steps_analyzed"])
        rm.dataloader_ms, rm.forward_ms = s["avg_dataloader_ms"], s["avg_forward_ms"]
        rm.backward_ms, rm.optimizer_ms = s["avg_backward_ms"], s["avg_optimizer_ms"]
        rm.step_cpu_ms = s["avg_step_cpu_ms"]
    which = 1 if len(aligned) <= 1 else 0  # single rank -> worst series (trend.py:46)
    din.trend_step = _trend_in(res, S_STEP * 2 + which, 0)
    din.trend_wait = _trend_in(res, S_WAIT * 2 + which, 0)
    din.trend_dl = _trend_in(res, S_DL * 2 + which, 0)
    diag = _abi.diag_json("tml_diag_step_time", din)
    if diag is not None:
        diag["issues"] = [dict(i, ranks=list(i["ranks"])) for i in diag["issues"]]
    return {"data": data, "diagnosis": diag, "global": step_time_global(aligned),
            "overview": step_time_overview(aligned)}


# ----------------------------------------------------------------------------- step memory
def step_memory_global(per_rank_means: Dict[str, Dict[str, float]]) -> Dict[str, Any]:
    """step_memory/model.py:322-412."""
    avg, med, worst = {}, {}, {}
    for name in ("peak_allocated_bytes", "peak_reserved_bytes"):
        vals = {k: float(v[name]) for k, v in per_rank_means.items()
                if v.get(name) is not None and math.isfinite(float(v[name]))}
        avg[name] = sum(vals.values()) / len(vals) if vals else None
        if not vals:
            med[name] = worst[name] = {"value": None, "idx": None}
            continue
        mv = statistics.median(vals.values())
        mk = min(vals, key=lambda k: (abs(vals[k] - mv), vals[k], int(k)))
        wk = max(vals, key=lambda k: (vals[k], -int(k)))
        med[name] = {"value": vals[mk], "idx": mk}
        worst[name] = {"value": vals[wk], "idx": wk}
    return {"average": avg, "median": med, "worst": worst}


def build_step_memory(out: ReduceOutput, gpu_total_bytes: Optional[float],
                      no_gpu_detected: bool = False) -> Dict[str, Any]:
    res = out.mem
    infos = out.infos
    have = [r for r in out.ranks if infos[r]["n_retained"] > 0]
    latest = max((infos[r]["latest_step"] for r in have), default=None)
    used = sorted(res.windows)
    n = int(res.n_common if used else 0)
    means = {str(r): {"peak_allocated_bytes": res.windows[r].m_sums[0] / n,
                      "peak_reserved_bytes": res.windows[r].m_sums[1] / n} for r in used} if n else {}
    # ranks that ever reported a step-memory row (loader.py:98-109)
    seen = len(have)
    din = _abi.MemDiagIn()
    din.steps_used = n
    din.window_size = int(out.window)
    din.completed_step = int(res.end_step or 0)
    din.ranks_seen = seen
    din.gpu_total_bytes = float(gpu_total_bytes) if gpu_total_bytes else 0.0
    din.n_metrics = 2 if n else 0
    which_series = ((S_ALLOC * 2, S_ALLOC * 2 + 1), (S_RESV * 2, S_RESV * 2 + 1))
    metrics = []
    for mi in range(din.n_metrics):
        m = din.metric[mi]
        m.n_ranks = len(used)
        for i, r in enumerate(used):
            m.ranks[i] = int(r)
            m.rank_peak[i] = float(res.windows[r].m_sums[2 + mi])
        med_s, worst_s = which_series[mi]
        m.trend_median = _trend_in(res, med_s, 1)
        m.trend_worst = _trend_in(res, worst_s, 1)
        m.points = n
        m.tail_first = res.tail_first[worst_s] if res.tail_first else float("nan")
        m.tail_last = res.tail_last[worst_s] if res.tail_last else float("nan")
    diag = _abi.diag_json("tml_diag_step_memory", din)
    for mi, name in enumerate(("peak_allocated", "peak_reserved")[: din.n_metrics]):
        sig = diag["metric_attribution"][name]
        metrics.append({
            "metric": name,
            "summary": {"window_size": int(out.window), "steps_used": n,
                        "median_peak": sig["median_peak_bytes"], "worst_peak": sig["worst_peak_bytes"],
                        "worst_rank": sig["worst_rank"], "skew_ratio": sig["skew_ratio"],
                        "skew_pct": sig["skew_pct"]},
            "coverage": {"expected_steps": int(out.window), "steps_used": n,
                         "completed_step": res.end_step, "world_size": seen,
                         "ranks_present": len(used), "incomplete": len(used) < seen},
        })
    return {
        "training_steps": (latest + 1) if latest is not None else 0,
        "latest_step_observed": latest,
        "gpu_total_bytes": gpu_total_bytes,
        "no_gpu_detected": bool(no_gpu_detected),
        "window": {"steps_first": res.start_step if n else None,
                   "steps_last": res.end_step if n else None, "n_steps": n,
                   "window_size": int(out.window), "global_ranks_seen": seen,
                   "global_ranks_used": len(used)},
        "metrics": metrics, "per_global_rank": means, "diagnosis": diag,
        "global": step_memory_global(means),
    }


# ----------------------------------------------------------------------------- process
def build_process(aggs: Dict[int, Dict[str, Any]]) -> Dict[str, Any]:
    """aggs[rank] = ProcAgg fields + ram_total + gpu_count."""
    din = _abi.ProcDiagIn()
    ranks = sorted(aggs)
    din.n_ranks = len(ranks)
    for i, r in enumerate(ranks):
        a = aggs[r]
        din.ranks[i] = int(r)
        for f, _ in _abi.ProcAgg._fields_:
            setattr(din.agg[i], f, a[f])
        din.ram_total[i] = float(a.get("ram_total", 0.0))
        din.gpu_count[i] = int(a.get("gpu_count", 0))
    return _abi.diag_json("tml_diag_process", din)


def proc_agg_dict(agg: _abi.ProcAgg, *, ram_total: float, gpu_count: int) -> Dict[str, Any]:
    d = {f: getattr(agg, f) for f, _ in _abi.ProcAgg._fields_}
    d["ram_total"] = float(ram_total)
    d["gpu_count"] = int(gpu_count)
    return d


# ----------------------------------------------------------------------------- driver
class SummaryEngine:
    """All three sections for the local engines of this process."""

    def __init__(self, engines, comm=None, *, exchange: str = "auto",
                 ram_total: Optional[float] = None, gpu_count: Optional[int] = None, native: bool = True):
        self.reducer = WindowReducer(engines, comm, exchange=exchange, native=native)
        self.engines = list(engines)
        self.comm = self.reducer.comm
        if ram_total is None:
            try:
                import psutil

                ram_total = float(psutil.virtual_memory().total)
            except Exception:
                ram_total = float(os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES"))
        self.ram_total = ram_total
        self.gpu_count = gpu_count

    def build(self, window: int = 10_000, proc_rows: int = 10_000, *, timings: bool = False) -> Dict[str, Any]:
        import torch

        gpu_count = self.gpu_count if self.gpu_count is not None else torch.cuda.device_count()
        if self.reducer._native_ok() and not timings:
            # one rank per process: stages, exchanges, rule engines and the section objects are
            # all native (csrc/tml_summary.cpp, tml_sections.cpp); the host parses one JSON
            from .reduce import NativeReduceOutput

            rows = max(1, int(proc_rows))
            o = self.reducer.run_native(max(1, int(window)), rows)
            res = self.engines[0].sections_json(o, self.ram_total, gpu_count, max(1, int(window)), rows)
            res["reduce"] = NativeReduceOutput(self.reducer, o, max(1, int(window)), rows)
            return res
        box: Dict[str, Any] = {}

        def _process(proc_aggs):
            # ram_total / gpu_count are per-host constants (psutil.virtual_memory().total,
            # torch.cuda.device_count()); single-node scope: identical on every rank
            aggs: Dict[int, Dict[str, Any]] = {}
            for r, a in proc_aggs.items():
                d = dict(a)
                d["ram_total"] = float(self.ram_total)
                d["gpu_count"] = int(gpu_count)
                aggs[r] = d
            box["aggs"] = aggs
            box["process"] = build_process(aggs)

        # the process rules need only the first exchange: they run under the K4 launch
        out = self.reducer.reduce(window, proc_rows=max(1, int(proc_rows)), overlap=_process,
                                  stage_timings=timings)
        if "aggs" not in box:  # native sequencing: no host window between the stages
            _process(out.proc_aggs)
        aggs = box["aggs"]
        with_gpu = [a for a in aggs.values() if a["n_gpu"] > 0]
        gpu_total = max((a["max_total"] for a in with_gpu), default=None)
        saw = [a for a in aggs.values() if a["n"] > 0]
        no_gpu = bool(saw) and not any(a["any_gpu_available"] for a in saw)
        return {
            "step_time": build_step_time(out),
            "step_memory": build_step_memory(out, gpu_total, no_gpu),
            "process": box["process"],
            "reduce": out,
        }


__all__ = ["SummaryEngine", "build_step_time", "build_step_memory", "build_process",
           "proc_agg_dict", "closest_rank_to_median", "step_time_global", "step_time_overview",
           "step_memory_global", "wait_avg_ms"]
