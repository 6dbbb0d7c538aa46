"""CPU, where the reference is installed in oracle/_ref: the bridge to the KEPT
payload builders.  Section dicts in the product's format (numbers from the oracle,
diagnoses from the native C++ engines) -> traceml_b200.reporting.to_reference_* ->
the reference's own build_*_payload / formatters == the golden payload JSON + card text."""
import os
import sys

import pytest

from helpers import (assert_struct, golden_cases, oracle_mem_rows, oracle_time_rows, plain,
                     proc_replay_for, step_replay_for)

reporting = pytest.importorskip("traceml_b200.reporting")
if not reporting.reference_available():
    pytest.skip("the reference is not installed in oracle/_ref", allow_module_level=True)

from oracle import step_memory_oracle, step_time_oracle  # noqa: E402
from test_native_diag_cpu import _agg_from_records  # noqa: E402
import replay  # noqa: E402
from traceml_b200 import sections  # noqa: E402

STEP = golden_cases("step")
PROC = golden_cases("process")


def _identities(n):
    return {r: {"global_rank": r, "local_rank": r, "node_rank": 0, "hostname": "b200-box",
                "local_world_size": n, "world_size": n} for r in range(n)}


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_time_payload_via_kept_builder(g):
    from traceml.reporting.sections.step_time.builder import build_step_time_payload
    from traceml.reporting.sections.step_time.formatter import format_step_time_section_text

    recs = step_replay_for(g)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, g["window"]), max_rows=g["window"])
    sec = {"data": {k: o["data"][k] for k in ("training_steps", "latest_step_observed", "aligned_summary",
                                              "aligned_window", "per_global_rank_summary", "max_rows")},
           "diagnosis": g["step_time"]["diagnosis"]}
    data, diag = reporting.to_reference_step_time(sec, _identities(g["ranks"]))
    payload = build_step_time_payload(data, diag)
    assert_struct(plain(payload), g["step_time"]["payload"], "payload", rel=0.0)
    assert format_step_time_section_text(payload) == g["step_time"]["text"]


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_memory_payload_via_kept_builder(g):
    from traceml.reporting.sections.step_memory.builder import build_step_memory_section_payload
    from traceml.reporting.sections.step_memory.formatter import format_step_memory_section_text

    recs = step_replay_for(g)
    ref = g["step_memory"]
    om = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=g["window"])
    sec = {"training_steps": om["training_steps"], "latest_step_observed": om["latest_step_observed"],
           "gpu_total_bytes": ref["gpu_total_bytes"], "no_gpu_detected": ref["no_gpu_detected"],
           "window": ref["window"],
           "metrics": [{"metric": m["metric"], "summary": m["summary"], "coverage": m["coverage"]}
                       for m in om["metrics"]],
           "per_global_rank": om["per_global_rank"], "diagnosis": ref["diagnosis"]}
    data, diag = reporting.to_reference_step_memory(sec, _identities(g["ranks"]))
    payload = build_step_memory_section_payload(data, diag)
    assert_struct(plain(payload), ref["payload"], "payload", rel=0.0)
    assert format_step_memory_section_text(payload) == ref["text"]


@pytest.mark.parametrize("g", PROC, ids=[g["case"] for g in PROC])
def test_process_payload_via_kept_builder(g):
    from traceml.reporting.sections.process.builder import build_process_payload
    from traceml.reporting.sections.process.formatter import format_process_section_text

    procs = proc_replay_for(g)
    aggs = {r: sections.proc_agg_dict(_agg_from_records(procs[r], g["max_rows"]),
                                      ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=g["ranks"])
            for r in procs}
    sec = sections.build_process(aggs)
    data, diag = reporting.to_reference_process(sec, _identities(g["ranks"]))
    payload = build_process_payload(data, diag)
    assert_struct(plain(payload), g["process"]["payload"], "payload", rel=1e-9)
    assert format_process_section_text(payload) == g["process"]["text"]


@pytest.mark.parametrize("scenario,pscenario,R,S,W", [("input_straggler", "normal", 4, 460, 10_000),
                                                      ("mem_imbalance", "overhang", 4, 260, 10_000),
                                                      ("balanced", "high_cpu", 1, 300, 128)])
def test_final_summary_envelope_equals_the_reference_report(tmp_path, scenario, pscenario, R, S, W):
    """End to end: the reference's FinalReportGenerator over its SQLite vs build_final_summary
    over this package's sections (engine double) -- same envelope keys, identical process /
    step_time / step_memory payloads, identical printed summary apart from the System card
    (the System section is outside this path)."""
    import torch
    from fake_engine import FakeEngine
    from traceml.reporting.final import build_final_report_generator

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_golden as mg

    recs = replay.make_step_replay(scenario, R, S, seed=5)
    procs = replay.make_proc_replay(pscenario, R, 200, seed=5)
    db = str(tmp_path / "telemetry")
    mg.build_db(db, step_records=recs, proc_records=procs)
    ref = build_final_report_generator(summary_window_rows=W).generate(db)
    se = sections.SummaryEngine([FakeEngine(recs[r], procs[r]) for r in range(R)],
                                ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)
    se.reducer.device = torch.device("cpu")
    res = se.build(W, W)
    ids = {r: {"global_rank": r, "local_rank": r, "node_rank": 0, "hostname": "b200-box",
               "local_world_size": R, "world_size": R} for r in range(R)}
    env = reporting.build_final_summary(res, ids)
    assert set(ref) <= set(env) and env["schema_version"] == ref["schema_version"] == 1.2
    for k in ("process", "step_time", "step_memory"):
        assert_struct(plain(env[k]), plain(ref[k]), k, rel=1e-12)

    def body(text):  # everything but the System card block
        lines = text.splitlines()
        i = next(n for n, l in enumerate(lines) if l.strip("| ").startswith("Process"))
        return lines[:3] + lines[i:]

    assert body(env["text"]) == body(ref["text"])
