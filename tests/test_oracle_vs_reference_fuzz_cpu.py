"""Oracle pin, widened: seeded random cases, the oracle against what the UNMODIFIED reference
computed for the same inputs, bit for bit.  The reference's outputs are stored in
tests/golden/fuzz.json.gz (tests/golden/make_fuzz_golden.py ran both sides and asserted them equal
before writing); here the oracle is re-run and compared with them."""
import gzip
import json
import os
import random

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FUZZ = os.path.join(HERE, "golden", "fuzz.json.gz")

SCENARIOS = ["balanced", "input_straggler", "compute_straggler", "straggler", "input_bound", "wait_heavy",
             "compute_bound", "ragged", "duplicates", "trend_worsening", "mem_creep_early", "mem_imbalance"]


def _cases(n, seed):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        out.append((rng.choice(SCENARIOS), rng.choice([1, 2, 3, 4, 5, 8]), rng.choice([60, 130, 260, 420]),
                    rng.randrange(1000), rng.choice([37, 100, 256, 10_000])))
    return out


STEP_CASES = _cases(10, 2026)
LIVE_CASES = _cases(8, 77)


def case_id(kind, scenario, ranks, steps, seed, window):
    return f"{kind}_{scenario}_r{ranks}_s{steps}_seed{seed}_w{window}"


def _load(name):
    with gzip.open(FUZZ, "rt") as fh:
        return json.load(fh)[name]


@pytest.mark.parametrize("scenario,ranks,steps,seed,window", STEP_CASES)
def test_final_summary_sections_oracle_equals_reference(scenario, ranks, steps, seed, window):
    """Everything tests/golden/make_golden.py::run_step_case compares, bit for bit."""
    from helpers import assert_struct, oracle_mem_rows, oracle_time_rows, plain, step_replay_for
    from oracle import step_memory_oracle, step_time_oracle

    g = _load(case_id("step", scenario, ranks, steps, seed, window))
    assert (g["scenario"], g["ranks"], g["steps"], g["seed"], g["window"]) == (scenario, ranks, steps, seed, window)
    recs = step_replay_for(g)
    # ---- step time: section data, diagnosis, public rollups
    ref_t = g["step_time"]
    assert ref_t["data"]["max_rows"] == window
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, window), max_rows=window)
    assert_struct(plain({k: o["data"][k] for k in ref_t["data"]}), ref_t["data"], "time.data", rel=0.0)
    assert_struct(plain(o["diagnosis"]), ref_t["diagnosis"], "time.diagnosis", rel=0.0)
    for k in ("average", "median", "worst"):
        assert_struct(plain(o["global"][k]), ref_t["payload"]["global"][k], f"time.global.{k}", rel=0.0)
    # ---- step memory: window, metrics, per-rank rows, diagnosis with attribution, rollups
    ref_m = g["step_memory"]
    om = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=window, gpu_total_bytes=None)
    w = ref_m["window"]
    assert om["training_steps"] == ref_m["training_steps"]
    assert om["window"]["global_ranks_seen"] == w["global_ranks_seen"]
    assert om["window"]["global_ranks_used"] == w["global_ranks_used"]
    assert len(om["window"]["steps"]) == w["n_steps"]
    if om["window"]["steps"]:
        assert (om["window"]["steps"][0], om["window"]["steps"][-1]) == (w["steps_first"], w["steps_last"])
    assert_struct(plain([{"metric": m["metric"], "summary": m["summary"], "coverage": m["coverage"]}
                         for m in om["metrics"]]), ref_m["metrics"], "mem.metrics", rel=0.0)
    assert_struct(plain(om["per_global_rank"]), ref_m["per_global_rank"], "mem.rows", rel=0.0)
    od, rd = plain(om["diagnosis"]), ref_m["diagnosis"]
    assert_struct(od["primary"], rd["primary"], "mem.primary", rel=0.0)
    assert_struct(od["issues"], rd["issues"], "mem.issues", rel=0.0)
    for mk, sig in rd["metric_attribution"].items():
        # ``device`` is the reference's majority label, tie-broken by Python set order
        # (model.py:122-127): not reproducible, not compared
        sig = {k: v for k, v in sig.items() if k != "device"}
        assert_struct({k: od["metric_attribution"][mk][k] for k in sig}, sig, f"mem.attr.{mk}", rel=0.0)
    if ref_m["payload"]["global"]:
        for k in ("average", "median", "worst"):
            assert_struct(plain(om["global"][k]), ref_m["payload"]["global"][k], f"mem.global.{k}", rel=0.0)


@pytest.mark.parametrize("scenario,ranks,steps,seed,window", LIVE_CASES)
def test_live_views_oracle_equals_reference(scenario, ranks, steps, seed, window):
    from helpers import assert_struct, plain
    from oracle import live_oracle
    import replay
    from test_live_cpu import mem_rows, wire_rows

    g = _load(case_id("live", scenario, ranks, steps, seed, window))
    t, m = g["time"], g["memory"]
    w = min(window, 400)
    assert t["window"] == m["window"] == w
    recs = replay.make_step_replay(scenario, ranks, steps, seed)
    assert replay.replay_digest(recs) == t["digest"] == m["digest"]
    rows = wire_rows(recs)
    cli = live_oracle.live_step_time(rows, window=w, include_series=True)
    dash = live_oracle.live_step_time(rows, window=w, include_series=False, include_rank_heatmap=True)
    assert_struct(plain(cli), t["cli"], "cli", rel=0.0)
    assert_struct(plain(dash), t["dashboard"], "dashboard", rel=0.0)
    o = live_oracle.live_step_memory(mem_rows(recs), window=w, gpu_available=m["gpu_available"])
    assert_struct(plain(o), m["result"], "memory", rel=0.0)
