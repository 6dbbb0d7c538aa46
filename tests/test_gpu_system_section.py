"""GPU: the System section on the device.

- records committed by k_sys_commit and bulk-loaded by tml_sys_load read back byte-identical,
  across a ring wrap;
- K6s (k_sys_reduce) equals oracle/system_oracle.py with ``==`` on every aggregate field, for every
  golden stream and for n = 1, 31, 32, 33, 10^4 + 1 over a wrapped ring and 10^5; its labels equal
  the goldens';
- the single-rank chained build with system samples: the section equals the oracle's and the Python
  driver's; back-to-back builds repeat it bit for bit; the other three sections are the same as
  before the samples were loaded; K6s is exactly one more launch when samples exist and none when
  they do not;
- a real training loop with ``TraceMLRuntime(sample_system=True)`` and the compatibility SQLite
  sink: final_summary()'s System payload equals the reference's ``SystemSummarySection`` over the
  database the same rows went to.
"""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import system_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN_DIR = os.path.join(HERE, "golden", "system")
GOLDENS = [json.load(open(os.path.join(GOLDEN_DIR, f))) for f in sorted(os.listdir(GOLDEN_DIR))
           if f.endswith(".json") and f != "INDEX.json"]

AGG_FIELDS = {  # SystemSummaryAgg key -> tml_sys_agg field (None columns: n_gpu == 0)
    "first_ts": "first_ts", "last_ts": "last_ts", "cpu_avg_percent": "cpu_avg", "cpu_peak_percent": "cpu_peak",
    "ram_avg_bytes": "ram_avg", "ram_peak_bytes": "ram_peak", "ram_total_bytes": "ram_total",
    "gpu_util_avg_percent": "gpu_util_avg", "gpu_util_peak_percent": "gpu_util_peak",
    "gpu_mem_avg_bytes": "gpu_mem_avg", "gpu_mem_peak_bytes": "gpu_mem_peak",
    "gpu_temp_avg_c": "gpu_temp_avg", "gpu_temp_peak_c": "gpu_temp_peak",
    "gpu_power_avg_w": "gpu_power_avg", "gpu_power_peak_w": "gpu_power_peak",
}
GPU_FIELDS = {"util_avg_percent": "util_avg", "util_peak_percent": "util_peak", "mem_avg_bytes": "mem_avg",
              "mem_peak_bytes": "mem_peak", "mem_total_bytes": "mem_total", "temp_avg_c": "temp_avg",
              "temp_peak_c": "temp_peak", "power_avg_w": "power_avg", "power_peak_w": "power_peak",
              "power_limit_w": "power_limit"}


@pytest.fixture(scope="module")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _engine(slots):
    from traceml_b200.engine import Engine

    return Engine(device=0, rank=0, world=1, ring_slots=1024, proc_slots=int(slots))


def _reduce(eng, rows):
    import torch

    s = torch.cuda.Stream()
    l0 = eng.launch_count
    eng.sys_reduce_launch(rows, int(s.cuda_stream))
    agg = eng.sys_reduce_collect()
    return agg, eng.launch_count - l0


def _assert_agg_equals_oracle(agg, sec, where=""):
    ag = sec["aggregate"]
    assert agg.n == ag["system_samples"], where
    if not agg.n:
        return
    for k, f in AGG_FIELDS.items():
        if ag[k] is None:
            assert agg.n_gpu == 0, (where, k)
            continue
        assert getattr(agg, f) == ag[k], (where, k, getattr(agg, f), ag[k])
    assert bool(agg.gpu_available) == ag["gpu_available"] and agg.gpu_count == ag["gpu_count"], where
    per = next(iter(sec["nodes"].values()))["per_gpu"]
    assert agg.n_gpus == len(per), where
    for i, q in per.items():
        for k, f in GPU_FIELDS.items():
            assert getattr(agg.gpu[int(i)], f) == q[k], (where, i, k, getattr(agg.gpu[int(i)], f), q[k])


# ----------------------------------------------------------------------------- ring
def test_commit_and_load_read_back_byte_identical(cuda):
    import torch

    raw = sc.random_raw(40, 5, seed=3)
    recs = sc.sys_records(raw)
    eng = _engine(24)
    try:
        s = torch.cuda.Stream()
        for i in range(10):  # through the commit kernel (record as a kernel argument) ...
            eng.sys_commit(recs[i], int(s.cuda_stream))
        s.synchronize()
        got = eng.sys_read(24)
        assert len(got) == 10 and eng.sys_count == 10
        assert b"".join(bytes(r) for r in got) == b"".join(bytes(recs[i]) for i in range(10))
        tail = (type(recs[0]) * 30)(*recs[10:40])  # ... then a bulk load that wraps the 24-slot ring
        eng.load_sys(tail)
        torch.cuda.synchronize()
        got = eng.sys_read(100)
        assert len(got) == 24 and eng.sys_count == 40
        assert b"".join(bytes(r) for r in got) == b"".join(bytes(recs[i]) for i in range(16, 40))
    finally:
        eng.close()


# ----------------------------------------------------------------------------- K6s
@pytest.mark.parametrize("g", GOLDENS, ids=[g["case"] for g in GOLDENS])
def test_k_sys_reduce_equals_oracle_and_labels_equal_goldens(cuda, g):
    import torch
    from oracle import system_oracle
    from traceml_b200 import sections

    raw = sc.make_raw(g["case"])
    rows = [sc.wire_row(s) for s in raw]
    eng = _engine(1024)
    try:
        if raw:
            eng.load_sys(sc.sys_records(raw))
            torch.cuda.synchronize()
        agg, launches = _reduce(eng, g["window"])
        assert launches == (1 if raw else 0)
        sec = system_oracle.system_section(rows, g["identity"], g["window"])
        _assert_agg_equals_oracle(agg, sec, g["case"])
        got = sections.build_system(agg, g["identity"])
        assert got["diagnosis"] == g["section"]["diagnosis"]
    finally:
        eng.close()


@pytest.mark.parametrize("n,G,slots,rows,adv", [
    (1, 8, 64, 10_000, False), (31, 3, 64, 10_000, False), (32, 16, 64, 10_000, True), (33, 1, 64, 10_000, False),
    (15_001, 8, 10_001, 10_001, True),   # 10^4 + 1 retained over a wrapped ring
    (100_000, 8, 100_000, 100_000, True),
])
def test_k_sys_reduce_equals_oracle_at_edges(cuda, n, G, slots, rows, adv):
    import torch
    from oracle import system_oracle

    raw = sc.random_raw(n, G, seed=n, adversarial=adv)
    eng = _engine(slots)
    try:
        eng.load_sys(sc.sys_records(raw))
        torch.cuda.synchronize()
        agg, launches = _reduce(eng, rows)
        assert launches == 1
        keep = min(n, slots, rows)
        sec = system_oracle.system_section([sc.wire_row(s) for s in raw[n - keep:]], sc.IDENTITY, keep)
        _assert_agg_equals_oracle(agg, sec, f"n={n}")
        again, _ = _reduce(eng, rows)  # the re-armed ticket: a second launch repeats bit for bit
        assert bytes(again) == bytes(agg)
    finally:
        eng.close()


# ----------------------------------------------------------------------------- chained build
W_BULK, S_BULK = 300_000, 300_000


def test_chained_build_with_system_samples(cuda):
    import torch

    import replay
    from oracle import system_oracle
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=S_BULK + 8, proc_slots=65_536)
    try:
        eng.load_steps(replay.make_step_replay("balanced", 1, S_BULK, seed=77)[0])
        eng.load_procs(replay.make_proc_replay("normal", 1, 20_000, seed=5)[0])
        torch.cuda.synchronize()
        se = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1,
                                    system_identity=sc.IDENTITY)
        l0 = eng.launch_count
        empty = se.build(W_BULK, 10_000)
        launches_empty = eng.launch_count - l0
        assert empty["system"]["diagnosis"]["primary"]["kind"] == "NO_DATA"
        raw_empty = bytes(empty.raw)
        raw = sc.random_raw(12_000, 8, seed=11, adversarial=True)
        eng.load_sys(sc.sys_records(raw))
        torch.cuda.synchronize()
        l0 = eng.launch_count
        res = se.build(W_BULK, 10_000)
        assert eng.launch_count - l0 - launches_empty == 1
        assert res["reduce"].fused_rows
        assert bytes(res.raw) == raw_empty  # the other three sections are untouched
        system = res["system"]
        repeat = [se.build(W_BULK, 10_000)["system"] for _ in range(2)]
        py = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1,
                                    system_identity=sc.IDENTITY, native=False).build(W_BULK, 10_000)
        assert system == py["system"] == repeat[0] == repeat[1]
    finally:
        eng.close()
    want = system_oracle.system_section([sc.wire_row(s) for s in raw[-10_000:]], sc.IDENTITY, 10_000)
    got = json.loads(json.dumps(system))
    assert got["aggregate"] == json.loads(json.dumps(want["aggregate"]))
    assert got["diagnosis"] == json.loads(json.dumps(want["diagnosis"]))


# ----------------------------------------------------------------------------- training loop
def test_training_loop_system_payload_equals_reference_section(cuda, tmp_path):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "traceml")):
        pytest.skip("oracle/_ref (the installed reference) is not present")
    os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    import torch

    import traceml_b200 as tml
    from helpers import plain
    from traceml_b200 import runtime
    from traceml_b200.compat import SQLiteCompatWriter
    from traceml_b200.runtime import TraceMLRuntime, reset_trace_session_state
    from traceml_b200.samplers import _identity_fields

    reset_trace_session_state(0)
    tml.init(mode="auto")
    eng = runtime.get_engine()
    torch.cuda.synchronize()
    eng.drain(); eng.proc_drain()
    eng.reset()  # the process engine may carry samples of an earlier runtime in this session
    db = str(tmp_path / "telemetry")
    writer = SQLiteCompatWriter(db, _identity_fields(), pid=os.getpid())
    rt = TraceMLRuntime(interval_sec=0.02, sinks=[writer], sample_system=True)
    rt.start()
    model = torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.ReLU(), torch.nn.Linear(512, 10)).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    ds = torch.utils.data.TensorDataset(torch.randn(32 * 60, 256), torch.randint(0, 10, (32 * 60,)))
    for x, y in torch.utils.data.DataLoader(ds, batch_size=32):
        with tml.trace_step(model):
            loss = torch.nn.functional.cross_entropy(model(x.to("cuda")), y.to("cuda"))
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    rt.stop()
    writer.close()
    assert eng.sys_count >= 2
    mine = tml.final_summary(window_rows=10_000)
    from traceml.reporting.sections.system import SystemSummarySection

    want = SystemSummarySection().build(db)
    got = plain(mine["system"])
    want_p = plain(want.payload)

    def close(a, b, path):
        if isinstance(b, dict):
            assert set(a) == set(b), (path, sorted(set(a) ^ set(b)))
            for k in b:
                close(a[k], b[k], f"{path}.{k}")
        elif isinstance(b, list):
            assert len(a) == len(b), path
            for i, (x, y) in enumerate(zip(a, b)):
                close(x, y, f"{path}[{i}]")
        elif isinstance(b, float) and not isinstance(b, bool):
            assert a == pytest.approx(b, rel=1e-12, abs=0.0), (path, a, b)
        else:
            assert a == b, (path, a, b)

    close(got, want_p, "system")
    assert got["diagnosis"]["status"] == want_p["diagnosis"]["status"]
    from traceml.reporting.sections.system.formatter import format_system_section_text

    assert format_system_section_text(mine["system"]) == want.text

