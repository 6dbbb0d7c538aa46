"""CPU: the oracle against the committed golden vectors (the reference's own
outputs, produced by tests/golden/make_golden.py)."""
import pytest

from oracle import process_oracle, step_memory_oracle, step_time_oracle
from helpers import (assert_struct, golden_cases, oracle_mem_rows, oracle_proc_rows,
                     oracle_time_rows, plain, proc_replay_for, step_replay_for, strip_device)

STEP = golden_cases("step")
PROC = golden_cases("process")


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_time_oracle_matches_reference(g):
    recs = step_replay_for(g)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, g["window"]), max_rows=g["window"])
    ref = g["step_time"]
    od = plain({k: o["data"][k] for k in ref["data"]})
    assert_struct(od, ref["data"], "data", rel=0.0)          # same op order -> bit exact
    assert_struct(plain(o["diagnosis"]), ref["diagnosis"], "diagnosis", rel=0.0)
    for k in ("average", "median", "worst"):
        assert_struct(plain(o["global"][k]), ref["payload"]["global"][k], f"global.{k}", rel=0.0)


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_memory_oracle_matches_reference(g):
    recs = step_replay_for(g)
    ref = g["step_memory"]
    o = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=g["window"])
    assert o["training_steps"] == ref["training_steps"]
    assert len(o["window"]["steps"]) == ref["window"]["n_steps"]
    assert o["window"]["global_ranks_used"] == ref["window"]["global_ranks_used"]
    assert_struct(plain([{"metric": m["metric"], "summary": m["summary"], "coverage": m["coverage"]}
                         for m in o["metrics"]]), ref["metrics"], "metrics", rel=0.0)
    assert_struct(plain(o["per_global_rank"]), ref["per_global_rank"], "rows", rel=0.0)
    od, rd = strip_device(plain(o["diagnosis"])), strip_device(ref["diagnosis"])
    assert_struct(od["primary"], rd["primary"], "primary", rel=0.0)
    assert_struct(od["issues"], rd["issues"], "issues", rel=0.0)
    if "step_memory_with_total" in g:
        t = g["step_memory_with_total"]
        o2 = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=g["window"],
                                                    gpu_total_bytes=t["gpu_total_bytes"])
        assert_struct(plain(o2["diagnosis"]["primary"]), t["diagnosis"]["primary"], "total.primary", rel=0.0)


@pytest.mark.parametrize("g", PROC, ids=[g["case"] for g in PROC])
def test_process_oracle_matches_reference(g):
    procs = proc_replay_for(g)
    o = process_oracle.process_section(oracle_proc_rows(procs, g["ranks"]), max_rows=g["max_rows"])
    ref = g["process"]
    od = plain(o["diagnosis"])
    assert_struct(od["primary"], ref["diagnosis"]["primary"], "primary", rel=1e-12)
    assert [i["kind"] for i in od["issues"]] == [i["kind"] for i in ref["diagnosis"]["issues"]]
    for oi, ri in zip(od["issues"], ref["diagnosis"]["issues"]):
        assert_struct(oi, ri, ri["kind"], rel=1e-12)


def test_reference_known_answers():
    """The reference's own fixtures (SURVEY 8c): tests/reporting/summary/test_step_time.py:138-177
    -- 1 rank, 2 steps, dl 1 / fwd 5 / bwd 10 / opt 4 / step 30 -> median total 31.0, 3 steps."""
    ev = {f"_traceml_internal:{n}": {"cpu": {"is_gpu": False, "duration_ms": v, "n_calls": 1}}
          for n, v in (("dataloader_next", 1.0), ("forward_time", 5.0), ("backward_time", 10.0),
                       ("optimizer_step", 4.0), ("step_time", 30.0))}
    rows = {0: [{"step": 2, "events": ev}, {"step": 1, "events": ev}]}
    o = step_time_oracle.step_time_section(rows, max_rows=10_000)
    assert o["data"]["training_steps"] == 3
    assert o["global"]["median"]["total_step_ms"]["value"] == 31.0
    assert o["data"]["aligned_window"]["steps_analyzed"] == 2
    assert o["diagnosis"]["primary"]["kind"] == "WARMUP"
    assert o["diagnosis"]["primary"]["reason"] == \
        "Only 2 steps per rank available; summary diagnosis requires 50."


def test_warmup_text_vector():
    """tests/diagnostics/test_step_time.py:263-298."""
    r = step_time_oracle.warmup_result(40, 50)
    assert r["primary"]["reason"] == "Only 40 steps per rank available; summary diagnosis requires 50."


def test_memory_alignment_vector():
    """tests/reporting/summary/test_step_memory.py:206-298 -- aligned window (2, 3),
    means 115.0 / 215.0."""
    rows = {0: [(1, 100.0, 200.0), (2, 110.0, 210.0), (3, 120.0, 220.0)],
            1: [(2, 111.0, 211.0), (3, 121.0, 221.0), (4, 131.0, 231.0)]}
    o = step_memory_oracle.step_memory_section(rows, window_size=2)
    assert o["window"]["steps"] == (2, 3)
    assert o["per_global_rank"]["0"]["peak_allocated_bytes"] == 115.0
    assert o["per_global_rank"]["0"]["peak_reserved_bytes"] == 215.0
