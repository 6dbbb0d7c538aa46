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


# ----------------------------------------------------------------------------- system
def system_node_label(identity: Dict[str, Any]) -> str:
    """SystemNodeIdentity.label (reporting/sections/system/loader.py:78-81)."""
    if identity.get("node_rank") is not None:
        return str(int(identity["node_rank"]))
    return str(int(identity.get("global_rank") or 0))


def build_system(agg: Optional[_abi.SysAgg], identity: Dict[str, Any]) -> Dict[str, Any]:
    """The System section of the engine's one node from the K6s aggregates: the cluster aggregate,
    ``nodes``, ``expected_nodes`` (loader.py:159-167, 300-359) and the diagnosis of the C++ rule
    engine (``tml_diag_system``).  ``agg`` None or empty: no samples, the reference's NO_DATA."""
    if agg is None:
        agg = _abi.SysAgg()
    label = system_node_label(identity)
    din = _abi.SysDiagIn()
    din.node_rank = int(identity["node_rank"]) if identity.get("node_rank") is not None else -1
    din.node_label = label.encode()[:31]
    din.agg = agg
    d = _abi.diag_json("tml_diag_system", din)
    n = int(agg.n)
    nodes: Dict[str, Any] = {}
    expected = 1
    if n:
        ident = {"label": label}
        ident.update({k: identity.get(k) for k in ("node_rank", "hostname", "global_rank", "local_rank",
                                                   "local_world_size", "world_size")})
        nodes[label] = {"identity": ident, "aggregate": dict(d["aggregate"]),
                        "per_gpu": {int(k): v for k, v in d["per_gpu"].items()}}
        world, lws = identity.get("world_size"), identity.get("local_world_size")
        if world and lws:
            expected = max(1, int(math.ceil(float(world) / float(lws))))
    return {"aggregate": d["aggregate"], "nodes": nodes, "expected_nodes": expected,
            "diagnosis": {"primary": d["primary"], "issues": d["issues"]}}


def multi_node_run(comm) -> bool:
    """Is the System section gathered across nodes?  Only when the run has more than one process
    and, by the launcher's environment, more than one node: ``ceil(WORLD_SIZE / LOCAL_WORLD_SIZE)
    > 1``.  Every rank reads the same two variables, so every rank takes the same branch of what
    is a collective."""
    if int(getattr(comm, "world", 1)) <= 1:
        return False
    try:
        world, lws = int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_WORLD_SIZE"])
    except (KeyError, ValueError):
        return False
    return lws > 0 and math.ceil(world / lws) > 1


def node_ident(identity: Dict[str, Any]) -> _abi.SysNodeIdent:
    """The record identity of a System source (``reporting.default_identity`` fields)."""
    i = _abi.SysNodeIdent()
    i.global_rank = int(identity.get("global_rank") or 0)
    i.local_rank = int(identity.get("local_rank") or 0)
    i.node_rank = int(identity["node_rank"]) if identity.get("node_rank") is not None else -1
    i.world_size = int(identity.get("world_size") or 0)
    i.local_world_size = int(identity.get("local_world_size") or 0)
    i.hostname = str(identity.get("hostname") or "").encode()[: _abi.TML_HOSTNAME_MAX - 1]
    return i


def _record_identity(rec: _abi.SysNodeRecord) -> Dict[str, Any]:
    i = rec.ident
    ident = {"node_rank": int(i.node_rank) if i.node_rank >= 0 else None,
             "hostname": i.hostname.decode("utf-8", "replace"), "global_rank": int(i.global_rank),
             "local_rank": int(i.local_rank), "local_world_size": int(i.local_world_size),
             "world_size": int(i.world_size)}
    return dict({"label": system_node_label(ident)}, **ident)


def build_system_cluster(host_records: Sequence[_abi.SysNodeRecord], cluster: _abi.SysClusterOut) -> Dict[str, Any]:
    """The System section of every node from the gathered records and K6m's result: the same
    shape as ``build_system``, with one entry per node in ``nodes`` (in the string order of their
    labels, loader.py:300-359), the cluster aggregate over all their samples, the reference's
    ``expected_nodes`` (loader.py:159-167) and the cluster-wide diagnosis of
    ``tml_diag_system_cluster``."""
    kept = [host_records[int(k)] for k in cluster.order[: int(cluster.n_nodes)]]
    idents = [_record_identity(r) for r in kept]
    by_label = sorted(zip(idents, kept), key=lambda p: p[0]["label"])
    din = (_abi.SysDiagIn * max(1, len(by_label)))()
    for k, (ident, rec) in enumerate(by_label):
        din[k].node_rank = ident["node_rank"] if ident["node_rank"] is not None else -1
        din[k].node_label = ident["label"].encode()[:31]
        din[k].agg = rec.agg
    d = _abi.diag_system_cluster(din, len(by_label), cluster.agg)
    nodes = {ident["label"]: {"identity": ident, "aggregate": d["nodes"][ident["label"]]["aggregate"],
                              "per_gpu": {int(k): v for k, v in d["nodes"][ident["label"]]["per_gpu"].items()}}
             for ident, _ in by_label}
    cands = {int(math.ceil(float(i["world_size"]) / float(i["local_world_size"])))
             for i in idents if i["world_size"] and i["local_world_size"]}
    expected = max(1, cands.pop()) if len(cands) == 1 else max(1, len(nodes))
    return {"aggregate": d["aggregate"], "nodes": nodes, "expected_nodes": expected,
            "diagnosis": {"primary": d["primary"], "issues": d["issues"]}}


# ----------------------------------------------------------------------------- driver
class SummaryEngine:
    """All three sections for the local engines of this process."""

    def __init__(self, engines, comm=None, *, exchange: str = "auto",
                 ram_total: Optional[float] = None, gpu_count: Optional[int] = None, native: bool = True,
                 system_identity: Optional[Dict[str, Any]] = None):
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
        self._unemitted: Optional[_abi.Sections] = None  # the last native build's sections
        # the System section has one source per node: the engine of local rank 0, whose system
        # ring the sampler fills; its node identity comes from the launcher's environment.  On one
        # node that is comm index 0; on several, every node leader reduces its own ring and the
        # records meet on comm index 0 (multi_node_run).
        self.system_identity = system_identity
        self._ident: Optional[Dict[str, Any]] = None
        self._no_system: Optional[Dict[str, Any]] = None
        self.multi_node = multi_node_run(self.comm)
        self._node_ident: Optional[Dict[str, Any]] = None

    def _leader_identity(self) -> Dict[str, Any]:
        if self._node_ident is None:
            from .reporting import default_identity

            self._node_ident = self.system_identity or default_identity(
                self.comm.index, max(1, int(self.comm.world)) * max(1, len(self.engines)))
        return self._node_ident

    def _system_launch(self, rows: int):
        """K6s beside the window pass on the engine holding the system ring; None (and nothing
        launched) when this process is not its node's source or its ring is empty."""
        eng = self.engines[0] if self.engines else None
        if self.multi_node:
            source = int(self._leader_identity().get("local_rank") or 0) == 0
        else:
            source = self.comm.index == 0
        if not source or not hasattr(eng, "sys_reduce_beside") or eng.sys_count == 0:
            return None
        eng.sys_reduce_beside(rows, _stream_of(self.reducer.device))
        return eng

    def _system_gather(self, eng) -> Optional[Dict[str, Any]]:
        """Every rank packs its node record in device memory (valid only on a node leader with
        samples); one all-gather brings them to comm index 0, which folds them (K6m), copies the
        records and the cluster rollup back in one transfer and runs the cluster rules.  None on
        every other rank."""
        import ctypes as C

        import torch

        if eng is not None:
            eng.sys_reduce_collect()  # ends the launch; the node's aggregates stay in HBM for the pack
        dev, world = self.reducer.device, int(self.comm.world)
        rec = C.sizeof(_abi.SysNodeRecord)
        mine = torch.empty(rec, dtype=torch.uint8, device=dev)
        gathered = torch.empty(world * rec + C.sizeof(_abi.SysClusterOut), dtype=torch.uint8, device=dev)
        stream = _stream_of(dev)
        ident = node_ident(self._leader_identity()) if eng is not None else None
        self.engines[0].sys_node_pack(ident, mine, stream)
        self.comm.all_gather_into(gathered[: world * rec], mine)
        if self.comm.index != 0:
            return None
        self.engines[0].sys_cluster_launch(gathered, world, stream)
        records, cluster = self.engines[0].sys_cluster_collect(world)
        if cluster.n_dup:
            import sys

            print(f"[TraceML] System section: {int(cluster.n_dup)} node record(s) repeat a node label; "
                  "each label keeps the record of its lowest global rank", file=sys.stderr)
        return build_system_cluster(records, cluster)

    def _system_section(self, eng) -> Optional[Dict[str, Any]]:
        if self.multi_node:
            return self._system_gather(eng)
        if self._ident is None:
            from .reporting import default_identity

            self._ident = self.system_identity or default_identity(
                0, max(1, int(self.comm.world)) * max(1, len(self.engines)))
        if eng is None:  # zero samples (NO_DATA): the same section every build
            if self._no_system is None:
                self._no_system = build_system(None, self._ident)
            return self._no_system
        return build_system(eng.sys_reduce_collect(), self._ident)

    def build(self, window: int = 10_000, proc_rows: int = 10_000, *, timings: bool = False) -> Dict[str, Any]:
        import torch

        gpu_count = self.gpu_count if self.gpu_count is not None else torch.cuda.device_count()
        if self.reducer._native_ok() and not timings:
            # one rank per process: stages, exchanges, rule engines and the section objects are
            # all native (csrc/tml_summary.cpp, tml_sections.cpp); the host parses one JSON
            from .reduce import NativeReduceOutput

            # The text is emitted from the result's own copy: on first access, or by the next build
            # while its window pass runs, whichever comes first -- so back-to-back builds keep the
            # JSON emitter out of the time the GPU waits for the host.
            rows = max(1, int(proc_rows))
            w = max(1, int(window))
            prev = self._unemitted
            seng = self._system_launch(rows)  # K6s beside the window pass; nothing without samples
            o = self.reducer.run_native(w, rows, prev=prev if prev is not None and prev._raw is None else None)
            red = NativeReduceOutput(self.reducer, o, w, rows)
            res = _abi.Sections(src=red._snap, args=_abi.SectionsArgs(float(self.ram_total), int(gpu_count), w, rows, 0))
            res["reduce"] = red
            res["system"] = self._system_section(seng)
            self._unemitted = res
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

        seng = self._system_launch(max(1, int(proc_rows)))
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
            "system": self._system_section(seng),
            "reduce": out,
        }


__all__ = ["SummaryEngine", "build_step_time", "build_step_memory", "build_process", "build_system",
           "build_system_cluster", "multi_node_run", "node_ident", "system_node_label",
           "proc_agg_dict", "closest_rank_to_median", "step_time_global", "step_time_overview",
           "step_memory_global", "wait_avg_ms"]
