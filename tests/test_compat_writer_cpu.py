"""CPU, where the reference is installed in oracle/_ref: a database written by traceml_b200.compat.SQLiteCompatWriter
is consumed by the reference's OWN final-report sections and yields the golden payloads
(the kept consumers keep working on our output)."""
import os
import sys

import pytest

REF_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
if os.path.isdir(REF_SRC) and REF_SRC not in sys.path:
    sys.path.append(REF_SRC)
pytest.importorskip("traceml.reporting.sections.step_time", reason="reference not importable here")

from helpers import assert_struct, load_golden, plain, proc_replay_for, step_replay_for  # noqa: E402
from traceml_b200 import records as rec_mod  # noqa: E402
import replay  # noqa: E402
from traceml_b200.compat import SQLiteCompatWriter  # noqa: E402


def _ident(r, n):
    return {"global_rank": r, "local_rank": r, "node_rank": 0, "hostname": "b200-box",
            "local_world_size": n, "world_size": n}


@pytest.mark.parametrize("case", ["input_straggler_r4", "duplicates_r2", "ragged_r4_w64", "mem_creep_confirmed_r4"])
def test_reference_sections_read_our_database(tmp_path, case):
    from traceml.reporting.sections.step_memory import StepMemorySummarySection
    from traceml.reporting.sections.step_time import StepTimeSummarySection

    g = load_golden(case)
    recs = step_replay_for(g)
    db = str(tmp_path / "telemetry")
    for r in sorted(recs):
        w = SQLiteCompatWriter(db, _ident(r, g["ranks"]), pid=1000 + r)
        w.write_step_time([rec_mod.step_record_to_wire(x, device=f"cuda:{r}") for x in recs[r]])
        w.write_step_memory([rec_mod.step_record_to_memory_wire(x, device=f"cuda:{r}") for x in recs[r]])
        w.close()
    res = StepTimeSummarySection(max_rows=g["window"]).build(db)
    assert_struct(plain(res.payload), g["step_time"]["payload"], "step_time.payload", rel=0.0)
    assert res.text == g["step_time"]["text"]
    mres = StepMemorySummarySection(window_size=g["window"]).build(db)
    assert_struct(plain(mres.payload), g["step_memory"]["payload"], "step_memory.payload", rel=0.0)


def test_reference_process_section_reads_our_database(tmp_path):
    from traceml.reporting.sections.process import ProcessSummarySection

    g = load_golden("proc_overhang_r4")
    procs = proc_replay_for(g)
    db = str(tmp_path / "telemetry")
    for r in sorted(procs):
        w = SQLiteCompatWriter(db, _ident(r, g["ranks"]))
        w.write_process([rec_mod.proc_record_to_wire(x, pid=1000 + r, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                                     gpu_count=g["ranks"], device_index=r) for x in procs[r]])
        w.close()
    res = ProcessSummarySection(max_process_rows=g["max_rows"]).build(db)
    assert_struct(plain(res.payload), g["process"]["payload"], "process.payload", rel=0.0)
    assert res.text == g["process"]["text"]


def test_system_rows_equal_the_reference_writer_and_feed_its_section(tmp_path):
    """f3: the host / NVML snapshot has the reference's wire schema (SystemSample.to_wire), our
    two system tables hold exactly what the reference's own projection writer would store, and the
    kept SystemSummarySection builds its card from our database."""
    import sqlite3

    from traceml.aggregator.sqlite_writers import system as ref_w
    from traceml.reporting.sections.system import SystemSummarySection
    from traceml.samplers.schema.system import GPUMetrics, SystemSample

    from traceml_b200.samplers import SystemProbe, SystemSampler

    row = SystemProbe().sample()  # no NVML here: CPU / RAM only, still the reference's keys
    ref_row = SystemSample(sample_idx=1, timestamp=0.0, cpu_percent=1.0, ram_used=2.0, ram_total=3.0,
                           gpu_available=False, gpu_count=0, gpus=[]).to_wire()
    assert set(row) == set(ref_row) and row["seq"] == 1 and row["ram_total"] > 0
    s = SystemSampler()
    s.sample(); s.sample()
    pay = s.collect_payload()
    assert pay["sampler"] == "SystemSampler" and len(pay["tables"]["SystemTable"]) == 1  # max_rows_per_flush = 1
    # synthetic 4-GPU snapshots through both writers
    rows = []
    for i in range(60):
        gpus = [GPUMetrics(util=50.0 + g + i % 7, mem_used=(40 + g) * 2.0 ** 30, mem_total=180 * 2.0 ** 30,
                           temperature=55.0 + g, power_usage=600.0 + 10 * g + i, power_limit=1000.0) for g in range(4)]
        rows.append(SystemSample(sample_idx=i + 1, timestamp=1000.0 + i, cpu_percent=30.0 + i % 5, ram_used=64e9,
                                 ram_total=512e9, gpu_available=True, gpu_count=4, gpus=gpus).to_wire())
    ours, theirs = str(tmp_path / "ours"), str(tmp_path / "theirs")
    w = SQLiteCompatWriter(ours, _ident(0, 4))
    w.write_system(rows)
    w.close()
    conn = sqlite3.connect(theirs)
    ref_w.init_schema(conn)
    env = dict(_ident(0, 4), rank=0, sampler="SystemSampler", timestamp=0.0, tables={"SystemTable": rows})
    ref_w.insert_rows(conn, ref_w.build_rows(env, 1))
    conn.commit(); conn.close()
    for table in ("system_samples", "system_gpu_samples"):
        a = sqlite3.connect(ours).execute(f"SELECT * FROM {table} ORDER BY id").fetchall()
        b = sqlite3.connect(theirs).execute(f"SELECT * FROM {table} ORDER BY id").fetchall()
        strip = lambda rr: [r[:1] + r[2:] for r in rr]  # recv_ts_ns differs  # noqa: E731
        assert strip(a) == strip(b) and len(a) > 0, table
    mine, ref = SystemSummarySection().build(ours), SystemSummarySection().build(theirs)
    assert_struct(plain(mine.payload), plain(ref.payload), "system.payload", rel=0.0)
    assert mine.text == ref.text and mine.payload.get("diagnosis")
