#!/usr/bin/env python
"""Generate tests/golden/fuzz.json.gz: seeded random cases through the UNMODIFIED reference.

Same recipe as make_golden.py / make_live_golden.py (which assert the oracle equal to the
reference, bit for bit, before anything is written), over the random case lists of
tests/test_oracle_vs_reference_fuzz_cpu.py.  Needs the reference installed into oracle/_ref:

    python tests/golden/make_fuzz_golden.py
"""
from __future__ import annotations

import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402  (puts ROOT and the reference on sys.path)
import make_live_golden as mlg  # noqa: E402
from test_oracle_vs_reference_fuzz_cpu import LIVE_CASES, STEP_CASES, case_id  # noqa: E402

OUT = os.path.join(HERE, "fuzz.json.gz")


def _step_fields(g):
    """Every reference output run_step_case compares the oracle with; the payload bodies other
    than their ``global`` rollups and the card text are left out (the oracle does not build them)."""
    t, m = g["step_time"], g["step_memory"]
    keep = {k: g[k] for k in ("case", "kind", "scenario", "ranks", "steps", "seed", "window", "digest")}
    keep["step_time"] = {"data": t["data"], "diagnosis": t["diagnosis"], "payload": {"global": t["payload"]["global"]}}
    keep["step_memory"] = {k: m[k] for k in ("training_steps", "window", "metrics", "per_global_rank", "diagnosis")}
    keep["step_memory"]["payload"] = {"global": m["payload"].get("global")}
    return keep


def main():
    out = {}
    for scenario, ranks, steps, seed, window in STEP_CASES:
        g = mg.run_step_case(f"fuzz_{scenario}", scenario, ranks, steps, seed, window)
        out[case_id("step", scenario, ranks, steps, seed, window)] = _step_fields(g)
    for scenario, ranks, steps, seed, window in LIVE_CASES:
        w = min(window, 400)
        out[case_id("live", scenario, ranks, steps, seed, window)] = {
            "time": mlg.run_live_case(f"fuzz_{scenario}", scenario, ranks, steps, seed, w),
            "memory": mlg.run_live_mem_case(f"fuzz_{scenario}", scenario, ranks, steps, seed, w, None)}
    with gzip.GzipFile(OUT, "wb", mtime=0) as fh:
        fh.write(json.dumps(out, sort_keys=True, separators=(",", ":")).encode())


if __name__ == "__main__":
    main()
