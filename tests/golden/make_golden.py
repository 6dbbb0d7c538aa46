#!/usr/bin/env python
"""Generate tests/golden/*.json from the UNMODIFIED reference.

Needs the unmodified reference installed into oracle/_ref (oracle/install_reference.py):

    python tests/golden/make_golden.py

For every case it
  1. builds the seeded replay records (traceml_b200.replay),
  2. projects them into a SQLite file with the reference's *own* projection
     writers (aggregator/sqlite_writers/{step_time,step_memory,process}.py),
  3. runs the reference sections' load -> diagnose -> build_payload,
  4. checks the oracle (oracle/*.py) against those outputs -- this is the
     oracle's parity pin -- and
  5. writes inputs' digest + the reference outputs as the golden vector.

The golden files are what the tests compare against wherever the reference
is not installed.
"""

from __future__ import annotations

import dataclasses
import json
import math
import os
import sqlite3
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

import numpy as np  # noqa: E402

from oracle import process_oracle, step_memory_oracle, step_time_oracle  # noqa: E402
from traceml_b200 import records as rec_mod  # noqa: E402
import replay  # noqa: E402

from traceml.aggregator.sqlite_writers import process as ref_proc_w  # noqa: E402
from traceml.aggregator.sqlite_writers import step_memory as ref_mem_w  # noqa: E402
from traceml.aggregator.sqlite_writers import step_time as ref_time_w  # noqa: E402
from traceml.reporting.sections.process import ProcessSummarySection  # noqa: E402
from traceml.reporting.sections.step_memory import StepMemorySummarySection  # noqa: E402
from traceml.reporting.sections.step_time import StepTimeSummarySection  # noqa: E402

# (name, scenario, ranks, steps, seed, window)
STEP_CASES = [
    ("balanced_r4", "balanced", 4, 260, 1, 10_000),
    ("input_straggler_r4", "input_straggler", 4, 460, 0, 10_000),
    ("compute_straggler_r4", "compute_straggler", 4, 260, 2, 10_000),
    ("straggler_r4", "straggler", 4, 260, 3, 10_000),
    ("input_bound_r2", "input_bound", 2, 260, 4, 10_000),
    ("wait_heavy_r8", "wait_heavy", 8, 260, 5, 10_000),
    ("compute_bound_r3", "compute_bound", 3, 260, 6, 10_000),
    ("warmup_r2", "warmup", 2, 40, 7, 10_000),
    ("ragged_r4", "ragged", 4, 300, 8, 10_000),
    ("ragged_r4_w64", "ragged", 4, 300, 8, 64),
    ("trend_worsening_r2", "trend_worsening", 2, 600, 9, 10_000),
    ("duplicates_r2", "duplicates", 2, 120, 10, 10_000),
    ("empty_rank_r3", "empty_rank", 3, 100, 11, 10_000),
    ("no_overlap_r2", "no_overlap", 2, 80, 12, 10_000),
    ("single_rank", "balanced", 1, 300, 13, 10_000),
    ("single_rank_wait", "wait_heavy", 1, 300, 14, 10_000),
    ("window_smaller_r4", "input_straggler", 4, 500, 15, 128),
    ("mem_creep_confirmed_r4", "mem_creep_confirmed", 4, 300, 16, 10_000),
    ("mem_creep_early_r2", "mem_creep_early", 2, 300, 17, 10_000),
    ("mem_imbalance_r4", "mem_imbalance", 4, 120, 18, 10_000),
    ("mem_pressure_r2", "mem_pressure", 2, 120, 19, 10_000),
    ("cpu_only_r1", "cpu_only", 1, 120, 20, 10_000),
    ("balanced_r7_odd", "balanced", 7, 210, 21, 10_000),
    ("balanced_r8_w100", "balanced", 8, 1500, 22, 100),
]

# (name, scenario, ranks, samples, seed, max_rows)
PROC_CASES = [
    ("proc_normal_r4", "normal", 4, 400, 1, 10_000),
    ("proc_very_high_r2", "very_high_gpu", 2, 200, 2, 10_000),
    ("proc_high_r2", "high_gpu", 2, 200, 3, 10_000),
    ("proc_overhang_r4", "overhang", 4, 200, 4, 10_000),
    ("proc_imbalance_r4", "imbalance", 4, 200, 5, 10_000),
    ("proc_high_rss_r2", "high_rss", 2, 200, 6, 10_000),
    ("proc_high_cpu_r1", "high_cpu", 1, 200, 7, 10_000),
    ("proc_no_gpu_r1", "no_gpu", 1, 100, 8, 10_000),
    ("proc_window_r2", "normal", 2, 500, 9, 128),
]


def _envelope(sampler: str, rank: int, world: int, rows):
    return {
        "rank": rank, "global_rank": rank, "local_rank": rank,
        "world_size": world, "local_world_size": world, "node_rank": 0,
        "hostname": "b200-box", "pid": 1000 + rank, "sampler": sampler,
        "timestamp": 0.0, "tables": {"t": rows},
    }


def build_db(path: str, step_records=None, proc_records=None):
    """Project replay records through the reference's own sqlite writers."""
    conn = sqlite3.connect(path)
    ref_time_w.init_schema(conn)
    ref_mem_w.init_schema(conn)
    ref_proc_w.init_schema(conn)
    recv = 1
    if step_records:
        world = len(step_records)
        for rank in sorted(step_records):
            recs = step_records[rank]
            trows = [rec_mod.step_record_to_wire(r, device=f"cuda:{rank}") for r in recs]
            mrows = [rec_mod.step_record_to_memory_wire(r, device=f"cuda:{rank}") for r in recs]
            ref_time_w.insert_rows(conn, ref_time_w.build_rows(
                _envelope("StepTimeSampler", rank, world, trows), recv))
            ref_mem_w.insert_rows(conn, ref_mem_w.build_rows(
                _envelope("StepMemorySampler", rank, world, mrows), recv))
            recv += 1
    if proc_records:
        world = len(proc_records)
        for rank in sorted(proc_records):
            rows = [rec_mod.proc_record_to_wire(
                        r, pid=1000 + rank, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                        gpu_count=world, device_index=rank)
                    for r in proc_records[rank]]
            ref_proc_w.insert_rows(conn, ref_proc_w.build_rows(
                _envelope("ProcessSampler", rank, world, rows), recv))
            recv += 1
    conn.commit()
    conn.close()


def plain(obj):
    """dataclasses / tuples / numpy -> JSON-friendly structures."""
    if dataclasses.is_dataclass(obj) and not isinstance(obj, type):
        return plain(dataclasses.asdict(obj))
    if isinstance(obj, dict):
        return {str(k): plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [plain(v) for v in obj]
    if isinstance(obj, (np.integer,)):
        return int(obj)
    if isinstance(obj, (np.floating,)):
        return float(obj)
    return obj


def assert_same(a, b, path="", rel=0.0):
    """Structural equality; floats exact unless ``rel`` > 0."""
    if isinstance(a, dict) and isinstance(b, dict):
        assert set(a) == set(b), f"{path}: keys {sorted(a)} != {sorted(b)}"
        for k in a:
            assert_same(a[k], b[k], f"{path}.{k}", rel)
    elif isinstance(a, list) and isinstance(b, list):
        assert len(a) == len(b), f"{path}: len {len(a)} != {len(b)}"
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{path}[{i}]", rel)
    elif isinstance(a, float) or isinstance(b, float):
        if a is None or b is None or isinstance(a, (str, bool)) or isinstance(b, (str, bool)):
            assert a == b, f"{path}: {a!r} != {b!r}"
        elif rel == 0.0:
            assert float(a) == float(b), f"{path}: {a!r} != {b!r}"
        else:
            assert math.isclose(float(a), float(b), rel_tol=rel, abs_tol=1e-300), \
                f"{path}: {a!r} !~ {b!r}"
    else:
        assert a == b, f"{path}: {a!r} != {b!r}"


def _strip_series(diag):
    return diag


def run_step_case(name, scenario, ranks, steps, seed, window):
    records = replay.make_step_replay(scenario, ranks, steps, seed)
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        build_db(db, step_records=records)

        # ---- reference: Step Time ----
        sec = StepTimeSummarySection(max_rows=window)
        data = sec.load(db)
        diag_in = sec.to_diagnosis_input(data)
        diag = sec.diagnose(diag_in)
        result = sec.build_payload(data, diag)
        ref_time = {
            "data": {
                "training_steps": data.training_steps,
                "latest_step_observed": data.latest_step_observed,
                "aligned_summary": plain(data.aligned_summary),
                "aligned_window": plain(data.aligned_window),
                "per_global_rank_summary": plain(data.per_global_rank_summary),
                "max_rows": data.max_rows,
            },
            "diagnosis": plain(diag) if diag is not None else None,
            "payload": plain(result.payload),
            "text": result.text,
        }

        # ---- reference: Step Memory ----
        msec = StepMemorySummarySection(window_size=window)
        mdata = msec.load(db)
        mdiag = msec.diagnose(msec.to_diagnosis_input(mdata))
        mres = msec.build_payload(mdata, mdiag)
        ref_mem = {
            "training_steps": mdata.training_steps,
            "latest_step_observed": mdata.latest_step_observed,
            "gpu_total_bytes": mdata.gpu_total_bytes,
            "no_gpu_detected": mdata.no_gpu_detected,
            "window": {
                "steps_first": (mdata.aligned_window.steps[0] if mdata.aligned_window.steps else None),
                "steps_last": (mdata.aligned_window.steps[-1] if mdata.aligned_window.steps else None),
                "n_steps": len(mdata.aligned_window.steps),
                "window_size": mdata.aligned_window.window_size,
                "global_ranks_seen": mdata.aligned_window.global_ranks_seen,
                "global_ranks_used": mdata.aligned_window.global_ranks_used,
            },
            "metrics": [{"metric": m.metric, "summary": plain(m.summary),
                         "coverage": plain(m.coverage)} for m in mdata.metrics],
            "per_global_rank": {k: plain(dict(v.metrics)) for k, v in mdata.per_global_rank.items()},
            "diagnosis": plain(mdiag),
            "payload": plain(mres.payload),
            "text": mres.text,
        }

    # ---- oracle pin: Step Time ----
    rows_by_rank = {r: rec_mod.records_to_time_rows(records[r], window) for r in records
                    if len(records[r])}
    o = step_time_oracle.step_time_section(rows_by_rank, max_rows=window)
    od = o["data"]
    assert_same(plain({k: od[k] for k in ref_time["data"]}), ref_time["data"], f"{name}.time.data")
    assert_same(plain(o["diagnosis"]), ref_time["diagnosis"], f"{name}.time.diag")
    g = ref_time["payload"]["global"]
    og = plain(o["global"])
    for k in ("average", "median", "worst"):
        assert_same(og[k], g[k], f"{name}.time.global.{k}")

    # ---- oracle pin: Step Memory ----
    mrows = {}
    for r in records:
        has = (records[r]["flags"] & rec_mod.FLAG_HAS_MEM) != 0
        mrows[r] = [(int(s), (float(a) if h else None), (float(v) if h else None))
                    for s, a, v, h in zip(records[r]["step"], records[r]["peak_alloc"],
                                          records[r]["peak_resv"], has)]
    om = step_memory_oracle.step_memory_section(mrows, window_size=window, gpu_total_bytes=None)
    assert om["training_steps"] == ref_mem["training_steps"], name
    assert om["window"]["global_ranks_seen"] == ref_mem["window"]["global_ranks_seen"], name
    assert om["window"]["global_ranks_used"] == ref_mem["window"]["global_ranks_used"], name
    assert len(om["window"]["steps"]) == ref_mem["window"]["n_steps"], name
    if om["window"]["steps"]:
        assert om["window"]["steps"][0] == ref_mem["window"]["steps_first"], name
        assert om["window"]["steps"][-1] == ref_mem["window"]["steps_last"], name
    assert_same(plain([{"metric": m["metric"], "summary": m["summary"], "coverage": m["coverage"]}
                       for m in om["metrics"]]), ref_mem["metrics"], f"{name}.mem.metrics")
    assert_same(plain(om["per_global_rank"]), ref_mem["per_global_rank"], f"{name}.mem.rows")
    odiag = plain(om["diagnosis"])
    rdiag = ref_mem["diagnosis"]
    assert_same(odiag["primary"], rdiag["primary"], f"{name}.mem.primary")
    assert_same(odiag["issues"], rdiag["issues"], f"{name}.mem.issues")
    for mk, sig in rdiag["metric_attribution"].items():
        osig = odiag["metric_attribution"][mk]
        # ``device`` is the reference's majority label, tie-broken by Python
        # set order (model.py:122-127) -> not reproducible, not compared.
        sig.pop("device", None)
        assert_same({k: osig[k] for k in sig}, sig, f"{name}.mem.attr.{mk}")
    if ref_mem["payload"].get("global"):
        for k in ("average", "median", "worst"):
            assert_same(plain(om["global"][k]), ref_mem["payload"]["global"][k],
                        f"{name}.mem.global.{k}")

    return {
        "case": name, "kind": "step", "scenario": scenario, "ranks": ranks,
        "steps": steps, "seed": seed, "window": window,
        "digest": replay.replay_digest(records),
        "step_time": ref_time, "step_memory": ref_mem,
    }


def run_step_memory_with_total(name, scenario, ranks, steps, seed, window):
    """Step-memory with gpu_total known (needs process rows in the same DB)."""
    records = replay.make_step_replay(scenario, ranks, steps, seed)
    procs = replay.make_proc_replay("normal", ranks, 50, seed)
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        build_db(db, step_records=records, proc_records=procs)
        msec = StepMemorySummarySection(window_size=window)
        mdata = msec.load(db)
        mdiag = msec.diagnose(msec.to_diagnosis_input(mdata))
    mrows = {r: [(int(s), float(a), float(v)) for s, a, v in
                 zip(records[r]["step"], records[r]["peak_alloc"], records[r]["peak_resv"])]
             for r in records}
    om = step_memory_oracle.step_memory_section(
        mrows, window_size=window, gpu_total_bytes=mdata.gpu_total_bytes)
    odiag, rdiag = plain(om["diagnosis"]), plain(mdiag)
    assert_same(odiag["primary"], rdiag["primary"], f"{name}.memtotal.primary")
    assert_same(odiag["issues"], rdiag["issues"], f"{name}.memtotal.issues")
    return {"gpu_total_bytes": mdata.gpu_total_bytes, "diagnosis": rdiag}


def run_proc_case(name, scenario, ranks, samples, seed, max_rows):
    procs = replay.make_proc_replay(scenario, ranks, samples, seed)
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        build_db(db, proc_records=procs)
        sec = ProcessSummarySection(max_process_rows=max_rows)
        data = sec.load(db)
        diag = sec.diagnose(sec.to_diagnosis_input(data))
        res = sec.build_payload(data, diag)
    ref = {
        "aggregate": plain(data.aggregate),
        "per_global_rank": plain(data.per_global_rank),
        "diagnosis": plain(diag),
        "payload": plain(res.payload),
        "text": res.text,
    }
    rows = {}
    for r, recs in procs.items():
        rows[r] = []
        for x in recs:
            w = rec_mod.proc_record_to_wire(x, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                            gpu_count=ranks, device_index=r)
            g = w["gpu"] or {}
            rows[r].append({
                "ts": w["ts"], "cpu": w["cpu"], "cpu_cores": w["cpu_cores"],
                "ram_used": w["ram_used"], "ram_total": w["ram_total"],
                "gpu_available": w["gpu_available"], "gpu_count": w["gpu_count"],
                "mem_used": g.get("mem_used"), "mem_reserved": g.get("mem_reserved"),
                "mem_total": g.get("mem_total")})
    o = process_oracle.process_section(rows, max_rows=max_rows)
    oagg = plain(o["data"]["aggregate"])
    ragg = dict(ref["aggregate"])
    ragg.pop("gpu_mem_reserved_overhang_ratio", None)  # never filled by the loader
    assert_same({k: oagg[k] for k in ragg}, ragg, f"{name}.agg", rel=1e-12)
    for r, pr in ref["per_global_rank"].items():
        opr = plain(o["data"]["per_global_rank"][int(r)])
        assert_same({k: opr[k] for k in pr if k in opr}, {k: pr[k] for k in pr if k in opr},
                    f"{name}.rank{r}", rel=1e-12)
    od = plain(o["diagnosis"])
    assert_same(od["primary"], ref["diagnosis"]["primary"], f"{name}.primary")
    assert len(od["issues"]) == len(ref["diagnosis"]["issues"]), name
    for oi, ri in zip(od["issues"], ref["diagnosis"]["issues"]):
        assert_same(oi, ri, f"{name}.issue.{ri['kind']}", rel=1e-12)
    return {"case": name, "kind": "process", "scenario": scenario, "ranks": ranks,
            "samples": samples, "seed": seed, "max_rows": max_rows,
            "digest": replay.replay_digest(procs), "process": ref}


def main():
    out_dir = HERE
    index = []
    for case in STEP_CASES:
        g = run_step_case(*case)
        if case[1].startswith("mem_"):
            g["step_memory_with_total"] = run_step_memory_with_total(*case)
        path = os.path.join(out_dir, f"{case[0]}.json")
        with open(path, "w") as fh:
            json.dump(g, fh, indent=1, sort_keys=True)
        t = g["step_time"]["diagnosis"]
        m = g["step_memory"]["diagnosis"]
        print(f"{case[0]:28s} time={t['primary']['kind'] if t else None!s:18s} "
              f"mem={m['primary']['kind']:16s} n={g['step_time']['data']['aligned_window']['steps_analyzed']}")
        index.append(case[0])
    for case in PROC_CASES:
        g = run_proc_case(*case)
        with open(os.path.join(out_dir, f"{case[0]}.json"), "w") as fh:
            json.dump(g, fh, indent=1, sort_keys=True)
        print(f"{case[0]:28s} proc={g['process']['diagnosis']['primary']['kind']}")
        index.append(case[0])
    with open(os.path.join(out_dir, "INDEX.json"), "w") as fh:
        json.dump({"cases": index, "reference": "traceopt-ai/traceml v0.2.15 @ a659c95"}, fh, indent=1)
    print(f"wrote {len(index)} golden cases")


if __name__ == "__main__":
    main()
