"""Shared test helpers (test infrastructure, may import oracle/)."""
from __future__ import annotations

import json
import math
import os
from typing import Any, Dict

import numpy as np

from traceml_b200 import records as rec_mod
import replay

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Floats produced from identical integer-ns inputs differ from the reference only by
# summation order (tree reduce on the GPU vs sequential Python): SURVEY 8(d) tolerance.
REL_TOL = 1e-9


def golden_cases(kind: str):
    with open(os.path.join(GOLDEN_DIR, "INDEX.json")) as fh:
        names = json.load(fh)["cases"]
    out = []
    for n in names:
        with open(os.path.join(GOLDEN_DIR, f"{n}.json")) as fh:
            g = json.load(fh)
        if g["kind"] == kind:
            out.append(g)
    return out


def load_golden(name: str) -> Dict[str, Any]:
    with open(os.path.join(GOLDEN_DIR, f"{name}.json")) as fh:
        return json.load(fh)


def plain(obj):
    if hasattr(obj, "to_dict") and not isinstance(obj, dict):  # traceml_b200._abi.Sections (lazy view)
        obj = obj.to_dict()
    if isinstance(obj, dict):
        return {str(k): plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [plain(v) for v in obj]
    if isinstance(obj, np.integer):
        return int(obj)
    if isinstance(obj, np.floating):
        return float(obj)
    return obj


def assert_struct(a, b, path="", rel=REL_TOL):
    """ints / strings / bools / None exact; floats within ``rel``."""
    if isinstance(a, dict) and isinstance(b, dict):
        assert set(a) == set(b), f"{path}: keys {sorted(set(a) ^ set(b))} differ"
        for k in a:
            assert_struct(a[k], b[k], f"{path}.{k}", rel)
    elif isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        assert len(a) == len(b), f"{path}: len {len(a)} != {len(b)}"
        for i, (x, y) in enumerate(zip(a, b)):
            assert_struct(x, y, f"{path}[{i}]", rel)
    elif isinstance(a, bool) or isinstance(b, bool) or a is None or b is None \
            or isinstance(a, str) or isinstance(b, str):
        assert a == b, f"{path}: {a!r} != {b!r}"
    elif isinstance(a, float) or isinstance(b, float):
        assert math.isclose(float(a), float(b), rel_tol=rel, abs_tol=1e-12), f"{path}: {a!r} !~ {b!r}"
    else:
        assert a == b, f"{path}: {a!r} != {b!r}"


def step_replay_for(g):
    recs = replay.make_step_replay(g["scenario"], g["ranks"], g["steps"], g["seed"])
    assert replay.replay_digest(recs) == g["digest"], "replay generator drifted from the golden inputs"
    return recs


def proc_replay_for(g):
    recs = replay.make_proc_replay(g["scenario"], g["ranks"], g["samples"], g["seed"])
    assert replay.replay_digest(recs) == g["digest"], "replay generator drifted from the golden inputs"
    return recs


def oracle_time_rows(records, window):
    return {r: rec_mod.records_to_time_rows(records[r], window) for r in records if len(records[r])}


def oracle_mem_rows(records):
    out = {}
    for r in records:
        has = (records[r]["flags"] & rec_mod.FLAG_HAS_MEM) != 0
        out[r] = [(int(s), (float(a) if h else None), (float(v) if h else None))
                  for s, a, v, h in zip(records[r]["step"], records[r]["peak_alloc"],
                                        records[r]["peak_resv"], has)]
    return out


def oracle_proc_rows(procs, ranks):
    rows = {}
    for r, recs in procs.items():
        rows[r] = []
        for x in recs:
            w = rec_mod.proc_record_to_wire(x, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                            gpu_count=ranks, device_index=r)
            g = w["gpu"] or {}
            rows[r].append({"ts": w["ts"], "cpu": w["cpu"], "cpu_cores": w["cpu_cores"],
                            "ram_used": w["ram_used"], "ram_total": w["ram_total"],
                            "gpu_available": w["gpu_available"], "gpu_count": w["gpu_count"],
                            "mem_used": g.get("mem_used"), "mem_reserved": g.get("mem_reserved"),
                            "mem_total": g.get("mem_total")})
    return rows


def strip_device(diag):
    """``device`` in step-memory attribution is a Python-set tie-break in the
    reference (model.py:122-127): not reproducible, never compared."""
    if diag and "metric_attribution" in diag:
        for v in diag["metric_attribution"].values():
            if isinstance(v, dict):
                v.pop("device", None)
    return diag


def build_vs_row_oracles(eng, recs, W, proc_rows=None):
    """One native single-rank build of ``eng`` (which retains ``recs``) with window ``W``; its
    step-time and step-memory sections must equal the row-level oracles'.  Returns the build."""
    from oracle import step_memory_oracle, step_time_oracle
    from traceml_b200 import sections

    got = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, proc_rows or W)
    o = step_time_oracle.step_time_section(oracle_time_rows({0: recs}, W), max_rows=W)
    g = got["step_time"]
    assert_struct(plain(g["data"]), plain({k: o["data"][k] for k in g["data"]}), "data")
    assert_struct(plain(g["diagnosis"]), plain(o["diagnosis"]), "diagnosis")
    for k in ("average", "median", "worst"):
        assert_struct(plain(g["global"][k]), plain(o["global"][k]), f"global.{k}")
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows({0: recs}), window_size=W,
                                                gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
    gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
    assert_struct(gd["primary"], od["primary"], "mem.primary")
    assert_struct(gd["issues"], od["issues"], "mem.issues")
    assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")
    return got
