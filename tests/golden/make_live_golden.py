#!/usr/bin/env python
"""Generate tests/golden/live/*.json from the UNMODIFIED reference's live
Step-Time computer (renderers/step_time/compute.py, StepCombinedComputer).

Needs the unmodified reference installed into oracle/_ref:

    python tests/golden/make_live_golden.py

Same recipe as make_golden.py: seeded replay -> the reference's own SQLite
projection writer -> ``StepCombinedComputer._compute_impl`` in both its modes
(CLI: series; dashboard: rank heat-map).  The oracle (oracle/live_oracle.py) is
asserted equal, bit for bit, before a vector is written.
"""

from __future__ import annotations

import json
import os
import sqlite3
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402  (puts ROOT and the reference on sys.path)

from oracle import live_oracle  # noqa: E402
from traceml_b200 import records as rec_mod  # noqa: E402
import replay  # noqa: E402

from traceml.renderers.step_memory.common import (  # noqa: E402
    StepMemoryMetricsDB, build_step_memory_combined_result)
from traceml.renderers.step_time.compute import StepCombinedComputer  # noqa: E402

# (name, scenario, ranks, steps, seed, window)
LIVE_CASES = [
    ("live_balanced_r4", "balanced", 4, 260, 1, 100),
    ("live_input_straggler_r4", "input_straggler", 4, 460, 0, 100),
    ("live_compute_straggler_r4", "compute_straggler", 4, 260, 2, 100),
    ("live_wait_heavy_r8", "wait_heavy", 8, 260, 5, 100),
    ("live_ragged_r4", "ragged", 4, 300, 8, 100),
    ("live_ragged_r4_w16", "ragged", 4, 300, 8, 16),
    ("live_duplicates_r2", "duplicates", 2, 120, 10, 100),
    ("live_empty_rank_r3", "empty_rank", 3, 100, 11, 100),
    ("live_no_overlap_r2", "no_overlap", 2, 80, 12, 100),
    ("live_single_rank", "balanced", 1, 300, 13, 100),
    ("live_short_r2", "warmup", 2, 40, 7, 100),
    ("live_odd_r7", "balanced", 7, 210, 21, 50),
    ("live_cpu_only_r1", "cpu_only", 1, 120, 20, 100),
    ("live_big_window_r8", "balanced", 8, 1500, 22, 300),
]


# (name, scenario, ranks, steps, seed, window, process scenario | None)
LIVE_MEM_CASES = [
    ("livemem_creep_r4", "mem_creep_confirmed", 4, 300, 16, 100, "normal"),
    ("livemem_imbalance_r4", "mem_imbalance", 4, 120, 18, 50, "normal"),
    ("livemem_ragged_r4", "ragged", 4, 300, 8, 100, None),
    ("livemem_ragged_r4_w16", "ragged", 4, 300, 8, 16, None),
    ("livemem_duplicates_r2", "duplicates", 2, 120, 10, 100, None),
    ("livemem_empty_rank_r3", "empty_rank", 3, 100, 11, 100, None),
    ("livemem_no_overlap_r2", "no_overlap", 2, 80, 12, 100, None),
    ("livemem_single_rank", "balanced", 1, 300, 13, 400, "normal"),
    ("livemem_cpu_only_r1", "cpu_only", 1, 120, 20, 100, None),
    ("livemem_cpu_only_nogpu_r1", "cpu_only", 1, 120, 20, 100, "no_gpu"),
    ("livemem_default_r8", "balanced", 8, 1500, 22, 400, "normal"),
    ("livemem_odd_r7", "mem_pressure", 7, 210, 21, 50, None),
]


def mem_rows(records):
    out = {}
    for r in records:
        has = (records[r]["flags"] & rec_mod.FLAG_HAS_MEM) != 0
        out[r] = [(int(s), (float(a) if h else None), (float(v) if h else None))
                  for s, a, v, h in zip(records[r]["step"], records[r]["peak_alloc"],
                                        records[r]["peak_resv"], has)]
    return out


def run_live_mem_case(name, scenario, ranks, steps, seed, window, proc_scenario):
    records = replay.make_step_replay(scenario, ranks, steps, seed)
    procs = replay.make_proc_replay(proc_scenario, ranks, 20, seed) if proc_scenario else None
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        mg.build_db(db, step_records=records, proc_records=procs)
        mdb = StepMemoryMetricsDB(db)
        with mdb.connect() as conn:
            ref = mg.plain(build_step_memory_combined_result(conn, db=mdb, window_size=window))
            gpu_available = mdb.detect_gpu_available(conn)
    for m in ref["metrics"]:
        m.pop("device", None)  # majority vote broken by set order (common.py:400-408)
    o = live_oracle.live_step_memory(mem_rows(records), window=window, gpu_available=gpu_available)
    mg.assert_same(mg.plain(o), ref, f"{name}.mem")
    return {"case": name, "kind": "live_step_memory", "scenario": scenario, "ranks": ranks,
            "steps": steps, "seed": seed, "window": window, "gpu_available": gpu_available,
            "digest": replay.replay_digest(records), "result": ref}


def run_live_case(name, scenario, ranks, steps, seed, window):
    records = replay.make_step_replay(scenario, ranks, steps, seed)
    out = {}
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        mg.build_db(db, step_records=records)
        comp = StepCombinedComputer(db, window_size=window)
        conn = sqlite3.connect(db)
        conn.row_factory = sqlite3.Row
        for mode, kw in (("cli", dict(include_series=True, include_rank_heatmap=False)),
                         ("dashboard", dict(include_series=False, include_rank_heatmap=True))):
            out[mode] = mg.plain(comp._compute_impl(conn, **kw))
        conn.close()
    rows_by_rank = {r: [rec_mod.step_record_to_wire(x, device=f"cuda:{r}") for x in records[r]]
                    for r in records}
    for mode, kw in (("cli", dict(include_series=True, include_rank_heatmap=False)),
                     ("dashboard", dict(include_series=False, include_rank_heatmap=True))):
        o = live_oracle.live_step_time(rows_by_rank, window=window, **kw)
        mg.assert_same(mg.plain(o), out[mode], f"{name}.{mode}")
    return {"case": name, "kind": "live_step_time", "scenario": scenario, "ranks": ranks,
            "steps": steps, "seed": seed, "window": window,
            "digest": replay.replay_digest(records), "cli": out["cli"], "dashboard": out["dashboard"]}


def main():
    dst = os.path.join(HERE, "live")
    os.makedirs(dst, exist_ok=True)
    names = []
    for case in LIVE_CASES:
        g = run_live_case(*case)
        with open(os.path.join(dst, case[0] + ".json"), "w") as f:
            json.dump(g, f, separators=(",", ":"))
        names.append(case[0])
        print("ok", case[0], g["cli"]["status_message"])
    mem_names = []
    for case in LIVE_MEM_CASES:
        g = run_live_mem_case(*case)
        with open(os.path.join(dst, case[0] + ".json"), "w") as f:
            json.dump(g, f, separators=(",", ":"))
        mem_names.append(case[0])
        print("ok", case[0], g["result"]["status_message"], len(g["result"]["metrics"]))
    with open(os.path.join(dst, "INDEX.json"), "w") as f:
        json.dump({"cases": names, "mem_cases": mem_names}, f, indent=1)


if __name__ == "__main__":
    main()
