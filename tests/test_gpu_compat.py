"""GPU, f1: records produced by the KERNELS on a real training loop are drained into the
compatibility SQLite (traceml_b200/compat.py) and consumed by the UNMODIFIED reference
(oracle/_ref): its three summary sections, its FinalReportGenerator (``final_summary.json`` of the
aggregator path) and ``traceml compare`` -- next to this engine's own in-process summary of the
same records (aggregator/sqlite_writers/step_time.py:172-187, database/database_sender.py:49-66)."""
import json
import os
import sys

import pytest
import torch

from helpers import plain

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def test_reference_consumers_read_device_fed_database(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if not os.path.isdir(os.path.join(REF, "traceml")):
        pytest.skip("oracle/_ref (the installed reference) is not present")
    os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    torch.cuda.set_device(0)
    import traceml_b200 as tml
    from traceml_b200 import runtime
    from traceml_b200.compat import SQLiteCompatWriter
    from traceml_b200.runtime import TraceMLRuntime, reset_trace_session_state
    from traceml_b200.samplers import _identity_fields

    reset_trace_session_state(0)
    tml.init(mode="auto")
    eng = runtime.get_engine()
    torch.cuda.synchronize()
    eng.drain(); eng.proc_drain()
    db = str(tmp_path / "telemetry")
    writer = SQLiteCompatWriter(db, _identity_fields(), pid=os.getpid())
    rt = TraceMLRuntime(interval_sec=0.02, sinks=[writer], sample_system=True)
    rt.start()
    model = torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.ReLU(), torch.nn.Linear(512, 10)).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    ds = torch.utils.data.TensorDataset(torch.randn(32 * 80, 256), torch.randint(0, 10, (32 * 80,)))
    for x, y in torch.utils.data.DataLoader(ds, batch_size=32):
        with tml.trace_step(model):
            x, y = x.to("cuda"), y.to("cuda")
            loss = torch.nn.functional.cross_entropy(model(x), y)
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    rt.stop()
    writer.close()
    mine = tml.final_summary(window_rows=10_000)          # this engine, from the HBM ring
    # ---- the reference's own consumers on the database the kernels' records went into
    from traceml.reporting.compare.command import compare_summaries
    from traceml.reporting.final import generate_summary
    from traceml.reporting.sections.process import ProcessSummarySection
    from traceml.reporting.sections.step_memory import StepMemorySummarySection
    from traceml.reporting.sections.step_time import StepTimeSummarySection

    st = StepTimeSummarySection(max_rows=10_000).build(db).payload
    sm = StepMemorySummarySection(window_size=10_000).build(db).payload
    pr = ProcessSummarySection().build(db).payload
    assert st["metadata"]["training_total_steps"] == 81 and st["metadata"]["global_ranks_used"] == 1
    assert st["diagnosis"]["status"] == mine["step_time"]["diagnosis"]["status"]
    assert sm["diagnosis"]["status"] == mine["step_memory"]["diagnosis"]["status"]
    assert pr["diagnosis"]["status"] is not None
    for roll in ("median", "worst"):   # same records, same arithmetic: the public rollups agree
        for metric, v in st["global"][roll].items():
            got = mine["step_time"]["global"][roll][metric]
            assert str(got["idx"]) == str(v["idx"]), (roll, metric)
            assert got["value"] == pytest.approx(v["value"], rel=1e-9, abs=1e-12), (roll, metric)
        for metric, v in sm["global"][roll].items():
            got = mine["step_memory"]["global"][roll][metric]
            assert str(got["idx"]) == str(v["idx"]) and got["value"] == pytest.approx(v["value"], rel=1e-12)
    # the aggregator-path artifact and `traceml compare` (kept CLI command) on it and on ours
    root = tmp_path / "session"
    ref_payload = generate_summary(db, session_root=str(root), print_to_stdout=False)
    assert (root / "final_summary.json").exists() and ref_payload["step_time"]["diagnosis"]["status"]
    assert ref_payload["system"] and ref_payload["system"].get("metadata") is not None   # f3 rows reached the System card
    # structural diff of the two final_summary documents: same keys, section by section, all the way down
    def tree(x):
        if isinstance(x, dict):
            return {k: tree(v) for k, v in sorted(x.items())}
        if isinstance(x, list):
            return [tree(x[0])] if x else []
        return type(x).__name__ if x is not None else "None"

    mine_p = plain(mine)
    for sec in ("step_time", "step_memory", "process"):
        a, b = tree(mine_p[sec]), tree(plain(ref_payload[sec]))
        for k in ("metadata", "diagnosis", "global", "groups", "units"):
            ak, bk = a.get(k), b.get(k)
            if isinstance(ak, dict) and isinstance(bk, dict):
                assert set(ak) == set(bk), (sec, k, sorted(set(ak) ^ set(bk)))
        assert set(a) == set(b), (sec, sorted(set(a) ^ set(b)))
    assert {"schema_version", "generated_at", "duration_s", "system", "process", "step_time", "step_memory", "text"} <= set(mine_p)
    ours_json = tmp_path / "ours_final_summary.json"
    ours_json.write_text(json.dumps(plain(mine)))
    cmp_payload = compare_summaries(root / "final_summary.json", ours_json, output=str(tmp_path / "cmp"),
                                    print_to_stdout=False)
    assert cmp_payload["text"] and os.path.exists(cmp_payload["artifacts"]["json"])
