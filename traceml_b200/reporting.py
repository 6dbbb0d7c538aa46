"""Bridge from the device-side sections to the KEPT reporting layer.

The reference's payload / card builders and ``FinalReportGenerator`` are kept,
not rebuilt (SURVEY section 2: ``reporting/sections/*/builder.py``,
``reporting/final.py``).  When the reference package ``traceml`` is importable,
``to_reference_*`` construct its own dataclasses
(``StepTimeSectionData`` + ``DiagnosticResult[StepDiagnosis]`` etc.) from our
section dicts and call its builders, so ``final_summary.json`` /
``final_summary.txt`` are produced by the unmodified reference code.  Without
the reference installed, ``build_final_summary`` returns the same numbers in a
plain envelope (no card text layout of its own).
"""

from __future__ import annotations

import os
import socket
import time
from typing import Any, Dict, Optional


def default_identity(rank: int, world: int) -> Dict[str, Any]:
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", str(world)) or world)
    return {
        "global_rank": int(rank),
        "local_rank": int(os.environ.get("LOCAL_RANK", str(rank % max(1, local_world)))),
        "node_rank": int(os.environ.get("GROUP_RANK", os.environ.get("NODE_RANK", "0")) or 0),
        "hostname": socket.gethostname(),
        "local_world_size": local_world,
        "world_size": int(world),
    }


_REF_TRIED = False


def reference_available() -> bool:
    """Is the KEPT reporting layer (the reference package ``traceml``) importable?  Looked for on
    ``sys.path`` first, then under ``$TRACEML_REFERENCE_PATH`` and the in-tree install
    ``<repo>/oracle/_ref`` (appended to ``sys.path``, never put in front of anything)."""
    global _REF_TRIED
    try:
        import traceml.reporting.sections.step_time.builder  # noqa: F401

        return True
    except Exception:
        pass
    if _REF_TRIED:
        return False
    _REF_TRIED = True
    import sys

    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for cand in (os.environ.get("TRACEML_REFERENCE_PATH"), os.path.join(here, "oracle", "_ref")):
        if cand and os.path.isdir(os.path.join(cand, "traceml")) and cand not in sys.path:
            sys.path.append(cand)
            os.environ.setdefault("TRACEML_LOGS_DIR", os.path.join("/tmp", "traceml_ref_logs"))
            try:
                import traceml.reporting.sections.step_time.builder  # noqa: F401

                return True
            except Exception:
                sys.path.remove(cand)
    return False


# ----------------------------------------------------------------------------- adapters
def _issues(items):
    from traceml.diagnostics.common import DiagnosticIssue

    return tuple(DiagnosticIssue(
        kind=i["kind"], status=i["status"], severity=i["severity"], summary=i["summary"],
        action=i["action"], metric=i.get("metric"), phase=i.get("phase"), score=i.get("score"),
        share_pct=i.get("share_pct"), skew_pct=i.get("skew_pct"),
        ranks=tuple(int(r) for r in i.get("ranks", ())), evidence=dict(i.get("evidence") or {}))
        for i in (items or ()))


def to_reference_step_time(sec: Dict[str, Any], identities: Dict[int, Dict[str, Any]]):
    """-> (StepTimeSectionData, Optional[DiagnosticResult[StepDiagnosis]])."""
    from traceml.diagnostics.common import DiagnosticResult
    from traceml.diagnostics.step_time.api import StepDiagnosis
    from traceml.reporting.sections.step_time.alignment import AlignedStepWindow
    from traceml.reporting.sections.step_time.loader import StepTimeSectionData
    from traceml.reporting.sections.step_time.model import GlobalRankIdentity, RankStepSummary

    d = sec["data"]
    mk = lambda s: RankStepSummary(**s)  # noqa: E731
    ids = {int(r): GlobalRankIdentity(**{k: v.get(k) for k in (
        "global_rank", "local_rank", "node_rank", "hostname", "local_world_size", "world_size")})
        for r, v in identities.items()}
    data = StepTimeSectionData(
        training_steps=d["training_steps"], latest_step_observed=d["latest_step_observed"],
        aligned_summary={int(r): mk(s) for r, s in d["aligned_summary"].items()},
        aligned_step_metrics={}, aligned_window=AlignedStepWindow(**d["aligned_window"]),
        per_global_rank_summary={int(r): mk(s) for r, s in d["per_global_rank_summary"].items()},
        per_global_rank_step_metrics={}, identities=ids, max_rows=d["max_rows"])
    diag = None
    if sec["diagnosis"] is not None:
        p = sec["diagnosis"]["primary"]
        diag = DiagnosticResult(
            primary=StepDiagnosis(severity=p["severity"], status=p["status"], reason=p["reason"],
                                  action=p["action"], kind=p["kind"], steps_used=p["steps_used"],
                                  worst_rank=p["worst_rank"], note=p["note"],
                                  confidence=p["confidence"]),
            issues=_issues(sec["diagnosis"]["issues"]),
            metric_attribution=sec["diagnosis"]["metric_attribution"])
    return data, diag


def to_reference_step_memory(sec: Dict[str, Any], identities: Dict[int, Dict[str, Any]]):
    from traceml.diagnostics.common import DiagnosticResult
    from traceml.diagnostics.step_memory import StepMemoryDiagnosis
    from traceml.renderers.step_memory.schema import (StepMemoryCombinedCoverage,
                                                      StepMemoryCombinedMetric,
                                                      StepMemoryCombinedSeries,
                                                      StepMemoryCombinedSummary)
    from traceml.reporting.sections.step_memory.loader import StepMemorySectionData
    from traceml.reporting.sections.step_memory.model import (StepMemoryAlignedWindow,
                                                              StepMemoryGlobalRankIdentity,
                                                              StepMemoryGlobalRankSummary)

    def ident(r):
        v = identities.get(int(r), {"global_rank": int(r)})
        return StepMemoryGlobalRankIdentity(**{k: v.get(k) for k in (
            "global_rank", "local_rank", "node_rank", "hostname", "local_world_size", "world_size")})

    metrics = [StepMemoryCombinedMetric(
        metric=m["metric"], device=None,
        series=StepMemoryCombinedSeries(steps=[], median=[], worst=[]),
        summary=StepMemoryCombinedSummary(**m["summary"]),
        coverage=StepMemoryCombinedCoverage(**m["coverage"])) for m in sec["metrics"]]
    rows = {k: StepMemoryGlobalRankSummary(identity=ident(k), metrics=dict(v))
            for k, v in sec["per_global_rank"].items()}
    w = sec["window"]
    data = StepMemorySectionData(
        training_steps=sec["training_steps"], latest_step_observed=sec["latest_step_observed"],
        metrics=metrics, gpu_total_bytes=sec["gpu_total_bytes"],
        no_gpu_detected=sec["no_gpu_detected"], per_global_rank=rows,
        aligned_window=StepMemoryAlignedWindow(steps=(), per_global_rank={},
                                               window_size=w["window_size"],
                                               global_ranks_seen=w["global_ranks_seen"]))
    p = sec["diagnosis"]["primary"]
    diag = DiagnosticResult(
        primary=StepMemoryDiagnosis(severity=p["severity"], status=p["status"], reason=p["reason"],
                                    action=p["action"], kind=p["kind"], metric=p["metric"],
                                    steps_used=p["steps_used"], worst_rank=p["worst_rank"],
                                    note=p["note"], confidence=p["confidence"]),
        issues=_issues(sec["diagnosis"]["issues"]),
        metric_attribution=sec["diagnosis"]["metric_attribution"])
    return data, diag


def to_reference_process(sec: Dict[str, Any], identities: Dict[int, Dict[str, Any]]):
    from traceml.diagnostics.common import DiagnosticResult
    from traceml.diagnostics.process import ProcessDiagnosis
    from traceml.reporting.sections.process.loader import ProcessSectionData
    from traceml.reporting.sections.process.model import PerRankProcessSummary, ProcessSummaryAgg

    agg = ProcessSummaryAgg(**sec["aggregate"])
    per = {}
    for r, v in sec["per_global_rank"].items():
        i = identities.get(int(r), {})
        per[int(r)] = PerRankProcessSummary(
            local_rank=i.get("local_rank"), world_size=i.get("world_size"),
            local_world_size=i.get("local_world_size"), node_rank=i.get("node_rank"),
            hostname=i.get("hostname"), **v)
    p = sec["primary"]
    diag = DiagnosticResult(
        primary=ProcessDiagnosis(severity=p["severity"], status=p["status"], reason=p["reason"],
                                 action=p["action"], kind=p["kind"], samples_used=p["samples_used"]),
        issues=_issues(sec["issues"]))
    return ProcessSectionData(aggregate=agg, per_global_rank=per), diag


def reference_payloads(res: Dict[str, Any], identities: Dict[int, Dict[str, Any]]) -> Dict[str, Any]:
    """Run the KEPT builders: {section: {"payload": ..., "text": ...}}."""
    from traceml.reporting.sections.process.builder import build_process_payload
    from traceml.reporting.sections.process.formatter import format_process_section_text
    from traceml.reporting.sections.step_memory.builder import build_step_memory_section_payload
    from traceml.reporting.sections.step_memory.formatter import format_step_memory_section_text
    from traceml.reporting.sections.step_time.builder import build_step_time_payload
    from traceml.reporting.sections.step_time.formatter import format_step_time_section_text

    out = {}
    d, g = to_reference_step_time(res["step_time"], identities)
    p = build_step_time_payload(d, g)
    out["step_time"] = {"payload": p, "text": format_step_time_section_text(p)}
    d, g = to_reference_step_memory(res["step_memory"], identities)
    p = build_step_memory_section_payload(d, g)
    out["step_memory"] = {"payload": p, "text": format_step_memory_section_text(p)}
    d, g = to_reference_process(res["process"], identities)
    p = build_process_payload(d, g)
    out["process"] = {"payload": p, "text": format_process_section_text(p)}
    return out


def build_final_summary(res: Dict[str, Any], identities: Optional[Dict[int, Dict[str, Any]]] = None
                        ) -> Dict[str, Any]:
    """The final_summary envelope: key set and formats of reporting/final.py:254-267
    (``schema_version 1.2, generated_at`` ISO-8601 UTC, ``duration_s, system, process,
    step_time, step_memory, text``).  With the reference importable the kept builders produce
    the section payloads and the kept ``final.py`` the combined text; the System section (NVML
    sampler: out of this path's scope) stays empty."""
    from datetime import datetime, timezone

    ranks = res["reduce"].ranks if "reduce" in res else []
    world = len(ranks) or 1
    identities = identities or {r: default_identity(r, world) for r in ranks}
    env: Dict[str, Any] = {"schema_version": 1.2, "generated_at": datetime.now(timezone.utc).isoformat(),
                           "duration_s": None, "system": {}, "engine": "traceml_b200"}
    if reference_available():
        from traceml.reporting import final as ref_final

        sec = reference_payloads(res, identities)
        for k in ("process", "step_time", "step_memory"):
            env[k] = dict(sec[k]["payload"])
        env["duration_s"] = ref_final._summary_duration_s(env["step_time"], env["process"], env["system"])
        env["text"] = ref_final._build_final_summary_text_from_sections(
            system_summary=env["system"], process_summary=env["process"],
            step_time_summary=env["step_time"], step_memory_summary=env["step_memory"])
    else:
        for k in ("process", "step_time", "step_memory"):
            env[k] = {kk: vv for kk, vv in res[k].items()} if isinstance(res[k], dict) else res[k]
        st = res["step_time"]["diagnosis"]
        sm = res["step_memory"]["diagnosis"]
        env["text"] = "\n".join([
            f"Step Time: {st['primary']['status'] if st else 'NO DATA'}"
            + (f" -- {st['primary']['reason']}" if st else ""),
            f"Step Memory: {sm['primary']['status']} -- {sm['primary']['reason']}",
            f"Process: {res['process']['primary']['status']} -- {res['process']['primary']['reason']}",
        ])
    return env


# ----------------------------------------------------------------------------- live views
def to_reference_step_combined(result: Dict[str, Any]):
    """``live.StepCombinedComputer`` result -> the reference's ``StepCombinedTimeResult``
    (renderers/step_time/schema.py:12-88), what the kept CLI renderer / dashboard consume."""
    from traceml.renderers.step_time.schema import (StepCombinedRankHeatmap, StepCombinedRankRow,
                                                    StepCombinedTimeCoverage, StepCombinedTimeMetric,
                                                    StepCombinedTimeResult, StepCombinedTimeSeries,
                                                    StepCombinedTimeSummary)

    metrics = [StepCombinedTimeMetric(
        metric=m["metric"], clock=m["clock"],
        series=StepCombinedTimeSeries(**m["series"]) if m["series"] else None,
        summary=StepCombinedTimeSummary(**m["summary"]),
        coverage=StepCombinedTimeCoverage(**m["coverage"])) for m in result["metrics"]]
    heat = None
    if result.get("rank_heatmap"):
        h = result["rank_heatmap"]
        heat = StepCombinedRankHeatmap(window_size=h["window_size"], steps_used=h["steps_used"],
                                       metric_keys=list(h["metric_keys"]),
                                       rows=[StepCombinedRankRow(rank=r["rank"], sums_ms=dict(r["sums_ms"]))
                                             for r in h["rows"]],
                                       sort_by=list(h["sort_by"]))
    return StepCombinedTimeResult(metrics=metrics, status_message=result["status_message"], rank_heatmap=heat)


def to_reference_step_memory_combined(result: Dict[str, Any]):
    """``live.StepMemoryCombinedComputer`` result -> ``StepMemoryCombinedResult``
    (renderers/step_memory/schema.py:8-72)."""
    from traceml.renderers.step_memory.schema import (StepMemoryCombinedCoverage, StepMemoryCombinedMetric,
                                                      StepMemoryCombinedResult, StepMemoryCombinedSeries,
                                                      StepMemoryCombinedSummary)

    metrics = [StepMemoryCombinedMetric(
        metric=m["metric"], device=m.get("device"),
        series=StepMemoryCombinedSeries(**m["series"]),
        summary=StepMemoryCombinedSummary(**m["summary"]),
        coverage=StepMemoryCombinedCoverage(**m["coverage"])) for m in result["metrics"]]
    return StepMemoryCombinedResult(metrics=metrics, status_message=result["status_message"])


class ReferenceComputerAdapter:
    """Drop-in for the ``_computer`` attribute of the kept renderers
    (renderers/step_time/renderer.py:56, step_memory/renderer.py:60): same ``compute_cli`` /
    ``compute_dashboard`` methods, reference dataclasses out, this package's live computer in."""

    def __init__(self, computer, convert):
        self._computer, self._convert = computer, convert

    def compute_cli(self):
        return self._convert(self._computer.compute_cli())

    def compute_dashboard(self):
        return self._convert(self._computer.compute_dashboard())


__all__ = ["to_reference_step_combined", "to_reference_step_memory_combined", "ReferenceComputerAdapter",
           "build_final_summary", "reference_payloads", "reference_available", "default_identity",
           "to_reference_step_time", "to_reference_step_memory", "to_reference_process"]
