"""GPU: the parity holes VERDICT r01 named.

(a) windows on both sides of the old reference-order-sum limit (2^17 rows), DISTINCT ranks, even R
    -- where ``closest_rank_to_median`` / argmax are decided on the last ulp of the per-rank sums --
    against the numpy oracle (oracle/fast_oracle.py, pinned == row-level oracle == reference);
(b) a5: per-step allocator peaks are the exact integers torch reports at the same point
    (reference: utils/step_memory.py:57,73-74);
(c) a9: every field of a process sample next to the UNMODIFIED reference's ProcessSampler
    (samplers/process_sampler.py:130-144,178-238) running in the same process;
(d) a1: stamp durations bracketed by CUDA events on both sides, SURVEY 8d tolerance
    (2 us + 1 %), and next to the reference's own CUDA-event timer path.
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

from helpers import assert_struct, plain, strip_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _engines(records, ring=None):
    from traceml_b200.engine import Engine

    R = len(records)
    out = []
    for r in range(R):
        e = Engine(device=0, rank=r, world=R, ring_slots=ring or (len(records[r]) + 8), proc_slots=64)
        e.load_steps(records[r])
        out.append(e)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------ (a)
@pytest.mark.parametrize("scenario,R,S,W", [
    ("balanced", 2, 131_072, 131_072), ("balanced", 2, 131_073, 131_073), ("balanced", 4, 200_000, 200_000),
    ("balanced", 2, 1_000_000, 1_000_000), ("input_straggler", 4, 140_000, 135_000),
    ("balanced", 8, 300_001, 300_001), ("balanced", 2, 60_000, 10_000), ("balanced", 6, 150_000, 140_000),
    ("ragged", 4, 150_000, 140_000), ("ragged", 2, 131_073, 131_073),   # offset + holey ranks: aligned K3e
])
def test_large_window_vs_numpy_oracle(cuda, scenario, R, S, W):
    import replay
    from oracle import fast_oracle
    from traceml_b200 import sections

    recs = replay.make_step_replay(scenario, R, S, seed=1000 + R)
    engines = _engines(recs)
    try:
        got = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R).build(W, W)
        ref_t = fast_oracle.step_time_section(recs, max_rows=W)
        ref_m = fast_oracle.step_memory_section(recs, window_size=W)
        gt, gm = got["step_time"], got["step_memory"]
        # integers, labels, rank ids: exact.  Floats: SURVEY 8d rel 1e-9 ...
        assert_struct(plain(gt["data"]["aligned_window"]), plain(ref_t["data"]["aligned_window"]), "window")
        assert_struct(plain(gt["diagnosis"]), plain(ref_t["diagnosis"]), "diagnosis")
        assert_struct(plain(gt["global"]), plain(ref_t["global"]), "global")
        assert_struct(plain(gt["overview"]), plain(ref_t["overview"]), "overview")
        # ... and the per-rank sums are BIT-exact (reference summation order reproduced on the GPU):
        # this is what makes every idx above safe, not luck
        assert plain(gt["data"]["aligned_summary"]) == plain(ref_t["data"]["aligned_summary"])
        assert plain(gt["data"]["per_global_rank_summary"]) == plain(ref_t["data"]["per_global_rank_summary"])
        assert plain(gm["per_global_rank"]) == plain(ref_m["per_global_rank"])      # exact integer sums
        assert_struct(plain(gm["global"]), plain(ref_m["global"]), "mem.global")
        gd, rd = strip_device(plain(gm["diagnosis"])), strip_device(plain(ref_m["diagnosis"]))
        assert_struct(gd["primary"], rd["primary"], "mem.primary")
        assert_struct(gd["issues"], rd["issues"], "mem.issues")
        # per-step series: ns->ms, median and max are exact operations -> bit equality
        red = got["reduce"]
        ser = red.time.series.cpu().numpy()
        np.testing.assert_array_equal(ser[:12], ref_t["_series"][:12])
        np.testing.assert_array_equal(red.mem.series.cpu().numpy()[12:16], ref_m["_series"])
    finally:
        for e in engines:
            e.close()


@pytest.mark.parametrize("scenario,S,W,ring,fused", [
    ("balanced", 300_000, 300_000, None, True), ("input_straggler", 450_000, 300_000, None, True),
    ("balanced", 400_000, 400_000, 250_000, True),      # ring wrapped: the window is what the ring retains
    ("duplicates", 200_000, 200_000, None, False),      # re-flushed step ids: not dense -> staged path
    ("balanced", 100_000, 100_000, None, False),        # below the bulk threshold: reference-order sums
])
def test_single_rank_bulk_path(cuda, scenario, S, W, ring, fused):
    """World of one, large window: ring -> series in one kernel (k_window_fused), accepted only if
    the window is dense.  Against the numpy oracle where step ids are unique, and bit for bit
    against the staged Python-sequenced path otherwise."""
    import replay
    from oracle import fast_oracle
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    recs = replay.make_step_replay(scenario, 1, S, seed=77)[0]
    slots = ring or (S + 8)
    kept = recs[-slots:]

    def run(native):
        eng = Engine(device=0, rank=0, world=1, ring_slots=slots, proc_slots=64)
        eng.load_steps(recs)
        torch.cuda.synchronize()
        try:
            res = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1,
                                         native=native).build(W, W)
            red = res["reduce"]
            ser = red.time.series.cpu().numpy().copy()
            mser = red.mem.series.cpu().numpy().copy()
            return res, ser, mser, bool(getattr(red, "fused_rows", False))
        finally:
            eng.close()

    got, ser, mser, was_fused = run(True)
    assert was_fused == fused
    staged, ser2, mser2, _ = run(False)
    np.testing.assert_array_equal(ser[:12], ser2[:12])
    np.testing.assert_array_equal(mser[12:16], mser2[12:16])
    for sec in ("step_time", "step_memory"):
        assert_struct(plain(got[sec]), plain(staged[sec]), f"fused == staged: {sec}", rel=1e-12 if fused else 0.0)
    if scenario != "duplicates":
        ref_t = fast_oracle.step_time_section({0: kept}, max_rows=W)
        ref_m = fast_oracle.step_memory_section({0: kept}, window_size=W)
        np.testing.assert_array_equal(ser[:12], ref_t["_series"][:12])
        np.testing.assert_array_equal(mser[12:16], ref_m["_series"])
        assert_struct(plain(got["step_time"]["data"]["aligned_window"]), plain(ref_t["data"]["aligned_window"]), "window")
        assert_struct(plain(got["step_time"]["data"]["aligned_summary"]), plain(ref_t["data"]["aligned_summary"]), "sums")
        assert_struct(plain(got["step_time"]["diagnosis"]), plain(ref_t["diagnosis"]), "diagnosis")
        assert_struct(plain(got["step_time"]["global"]), plain(ref_t["global"]), "global")
        assert plain(got["step_memory"]["per_global_rank"]) == plain(ref_m["per_global_rank"])
        gd, rd = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(ref_m["diagnosis"]))
        assert_struct(gd["primary"], rd["primary"], "mem.primary")


# ------------------------------------------------------------------------------------ (b)
def test_step_memory_peaks_are_torch_exact(cuda):
    """a5: peak_alloc / peak_resv of every step == torch.cuda.max_memory_allocated / reserved
    read at the end of that step (the reference resets at step entry and reads at step exit)."""
    import traceml_b200 as traceml
    from traceml_b200 import runtime
    from traceml_b200.runtime import reset_trace_session_state

    reset_trace_session_state(0)
    traceml.init(mode="auto")
    eng = runtime.get_engine()
    torch.cuda.synchronize()
    eng.drain()
    model = torch.nn.Sequential(torch.nn.Linear(512, 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 16)).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    expect = []
    for i in range(12):
        x = torch.randn(64 * (1 + i % 4), 512)
        y = torch.randint(0, 16, (x.shape[0],))
        with traceml.trace_step(model):
            xd, yd = x.to("cuda"), y.to("cuda")
            scratch = torch.empty((1 + (i * 7) % 5) << 20, dtype=torch.uint8, device="cuda")  # varies the peak
            loss = torch.nn.functional.cross_entropy(model(xd), yd)
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            del scratch
            expect.append((torch.cuda.max_memory_allocated(0), torch.cuda.max_memory_reserved(0)))
    torch.cuda.synchronize()
    recs, _ = eng.drain()
    assert len(recs) == 12
    assert [(int(a), int(b)) for a, b in zip(recs["peak_alloc"], recs["peak_resv"])] == expect
    assert len({a for a, _ in expect}) > 2, "the test must see different peaks in different steps"
    # and the wire row carries them as the reference does: float of the exact integer
    from traceml_b200.records import step_record_to_memory_wire

    w = step_record_to_memory_wire(recs[3], device="cuda:0")
    assert w["peak_alloc"] == float(expect[3][0]) and w["peak_resv"] == float(expect[3][1])


# ------------------------------------------------------------------------------------ (c)
def _reference():
    if not os.path.isdir(os.path.join(REF, "traceml")):
        pytest.skip("oracle/_ref (the installed reference) is not present")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")


def test_process_sample_fields_vs_reference_sampler(cuda):
    """a9, Python probe: same psutil estimators and allocator counters as the reference's
    ProcessSampler, sampled back to back in one process."""
    _reference()
    from traceml.samplers.process_sampler import ProcessSampler as RefProcessSampler

    from traceml_b200.engine import Engine
    from traceml_b200.samplers import ProcessProbe, drain_to_wire

    keep = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")  # something to report
    eng = Engine(device=0, ring_slots=64, proc_slots=256)
    ref, mine = RefProcessSampler(), ProcessProbe()
    t_end = time.perf_counter() + 0.3
    while time.perf_counter() < t_end:   # burn CPU so cpu_percent has something to measure
        sum(range(2000))
    ref.sample()
    mine.sample(eng)
    torch.cuda.synchronize()
    rrow = dict(list(ref.db.get_table("ProcessTable"))[-1])
    out = drain_to_wire(eng)
    assert len(out["process"]) == 1
    m = out["process"][0]
    assert set(m) == set(rrow), (sorted(m), sorted(rrow))
    assert m["pid"] == rrow["pid"] and m["cpu_cores"] == rrow["cpu_cores"]
    assert m["ram_total"] == rrow["ram_total"] and m["ram_total"] > 0
    assert m["gpu_available"] is True and rrow["gpu_available"] is True
    assert m["gpu_count"] == rrow["gpu_count"] == torch.cuda.device_count()
    assert set(m["gpu"]) == set(rrow["gpu"])
    # allocator counters: nothing allocates between the two samples -> exact
    assert m["gpu"]["mem_used"] == rrow["gpu"]["mem_used"] and m["gpu"]["mem_used"] >= float(64 << 20)
    assert m["gpu"]["mem_reserved"] == rrow["gpu"]["mem_reserved"]
    assert m["gpu"]["mem_total"] == rrow["gpu"]["mem_total"]
    assert m["gpu"]["device"] == rrow["gpu"]["device"] == 0
    # RSS read twice a few hundred microseconds apart
    assert abs(m["ram_used"] - rrow["ram_used"]) <= 8 << 20
    # both are psutil.Process.cpu_percent(interval=None) of the same process, windows ~equal
    assert m["cpu"] > 20.0 and rrow["cpu"] > 20.0 and abs(m["cpu"] - rrow["cpu"]) < 60.0
    del keep
    eng.close()


def test_native_sampler_fields_vs_psutil(cuda):
    """a9, native 1 kHz thread: RSS / allocator counters / total / cores equal the reference's
    sources; cpu_pct is the same estimator psutil uses -- (process user+sys CPU time delta) /
    (wall delta) x 100, not normalised by core count -- taken over the sampler's own period, so
    its WINDOW MEAN is compared with psutil over the same window.  Rows are taken as the wire
    rows the runtime hands to its sinks (samplers/schema/process.py:139-150)."""
    import psutil

    import traceml_b200 as traceml
    from traceml_b200 import runtime
    from traceml_b200.runtime import TraceMLRuntime

    traceml.init(mode="auto")
    eng = runtime.get_engine()
    torch.cuda.synchronize()
    eng.proc_drain()
    proc = psutil.Process(os.getpid())
    keep = torch.empty(32 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    rt = TraceMLRuntime(interval_sec=0.05, native_process_hz=500.0,
                        sinks=[lambda kind, r: rows.extend(r) if kind == "process" else None])
    proc.cpu_percent(interval=None)
    rt.start()
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < 0.8:
        sum(range(5000))                 # one busy Python thread: ~100 % of one core
    ps_cpu = proc.cpu_percent(interval=None)
    used, resv = torch.cuda.memory_allocated(0), torch.cuda.memory_reserved(0)
    rss = proc.memory_info().rss
    rt.stop()
    torch.cuda.synchronize()
    assert len(rows) > 200, len(rows)
    last = rows[-1]
    assert last["gpu"]["mem_used"] == float(used) and last["gpu"]["mem_reserved"] == float(resv)
    total = torch.cuda.get_device_properties(0).total_memory
    assert abs(last["gpu"]["mem_total"] - total) < (2 << 30)   # cudaMemGetInfo total vs device property
    assert last["cpu_cores"] == (psutil.cpu_count(logical=True) or 0)
    assert last["ram_total"] == float(psutil.virtual_memory().total)
    assert last["gpu_count"] == torch.cuda.device_count() and last["gpu_available"] is True
    assert last["pid"] == os.getpid()
    assert abs(last["ram_used"] - rss) <= 16 << 20
    seqs = [r["seq"] for r in rows]
    assert seqs == list(range(seqs[0], seqs[0] + len(seqs)))
    # window mean of the native estimator vs psutil over (almost) the same window
    mean_native = float(np.mean([r["cpu"] for r in rows[5:]]))
    assert abs(mean_native - ps_cpu) < 35.0, (mean_native, ps_cpu)
    assert mean_native > 50.0
    del keep


# ------------------------------------------------------------------------------------ (d)
def _spin_matmul(a, k):
    for _ in range(k):
        a = a @ a
        a = a / a.norm()
    return a


def test_stamp_bracketed_by_cuda_events(cuda):
    """a1: event_inner <= stamp <= event_outer, each within SURVEY 8d's 2 us + 1 %.

    The stamp kernels and the CUDA events are all in-stream timestamps; an event recorded
    OUTSIDE the stamp pair must see at least the stamp duration, one recorded INSIDE at most.
    The measured deltas travel in the assertion messages."""
    from traceml_b200.engine import Engine

    eng = Engine(device=0, ring_slots=1024)
    s = torch.cuda.current_stream()
    a = torch.randn(1024, 1024, device="cuda")
    a = _spin_matmul(a, 3)
    evs, n = [], 300
    for step in range(1, n + 1):
        eo0, eo1, ei0, ei1 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
        eo0.record()
        slot = eng.phase_begin(2, s.cuda_stream)
        ei0.record()
        a = _spin_matmul(a, 1 + step % 5)
        ei1.record()
        assert eng.phase_end(2, slot, s.cuda_stream) == 0
        eo1.record()
        evs.append((eo0, eo1, ei0, ei1))
        assert eng.step_commit(step, 0, 0, 0, 0.0, s.cuda_stream) == 0
        if step % 64 == 0:
            torch.cuda.synchronize()   # keep the host from running far ahead: gaps stay physical
    torch.cuda.synchronize()
    recs, dropped = eng.drain()
    assert dropped == 0 and len(recs) == n
    outer = np.array([e[0].elapsed_time(e[1]) * 1000.0 for e in evs])
    inner = np.array([e[2].elapsed_time(e[3]) * 1000.0 for e in evs])
    stamp = recs["dur_ns"][:, 2].astype(np.float64) / 1000.0
    tol = 2.0 + 0.01 * stamp
    hist = {"n": n, "unit": "us",
            "outer_minus_stamp": np.percentile(outer - stamp, [0, 5, 50, 95, 99, 100]).tolist(),
            "stamp_minus_inner": np.percentile(stamp - inner, [0, 5, 50, 95, 99, 100]).tolist(),
            "outer_minus_inner": np.percentile(outer - inner, [0, 5, 50, 95, 99, 100]).tolist(),
            "stamp_us": np.percentile(stamp, [0, 50, 100]).tolist(), "percentiles": [0, 5, 50, 95, 99, 100]}
    assert (stamp <= outer + tol).all(), hist
    assert (stamp >= inner - tol).all(), hist
    # means over >= 100 steps: the stamp mean lies inside the bracket means, 0.5 %
    assert inner.mean() * 0.995 - 2.0 <= stamp.mean() <= outer.mean() * 1.005 + 2.0, hist
    eng.close()


def test_phase_timers_next_to_the_reference_event_path(cuda):
    """a1/a7 side by side: the UNMODIFIED reference's timed_region (CUDA-event pairs resolved by
    its StepTimeSampler) nested immediately inside this engine's region, 200 steps.  Per phase
    and step the reference's figure is bracketed: ref <= ours + tol (it is the inner pair)."""
    _reference()
    import traceml.utils.timing as rt
    from traceml.runtime.state import reset_trace_session_state as ref_reset
    from traceml.samplers.step_time_sampler import StepTimeSampler as RefStepTimeSampler
    from traceml.utils.flush_buffers import flush_step_events as ref_flush

    from traceml_b200.engine import Engine

    ref_reset(0)
    eng = Engine(device=0, ring_slots=1024)
    s = torch.cuda.current_stream()
    a = torch.randn(1024, 1024, device="cuda")
    model = torch.nn.Linear(2, 2)
    sampler = RefStepTimeSampler()
    n = 200
    names = {2: "_traceml_internal:forward_time", 3: "_traceml_internal:backward_time"}
    for step in range(1, n + 1):
        for ph, name in names.items():
            slot = eng.phase_begin(ph, s.cuda_stream)
            with rt.timed_region(name, scope="step", use_gpu=True):
                a = _spin_matmul(a, 1 + (step + ph) % 4)
            eng.phase_end(ph, slot, s.cuda_stream)
        eng.step_commit(step, 0, 0, 0, 0.0, s.cuda_stream)
        ref_flush(model, step)
        if step % 50 == 0:
            torch.cuda.synchronize()
            sampler.sample()
    torch.cuda.synchronize()
    sampler.sample()
    recs, _ = eng.drain()
    rows = [dict(r) for r in sampler.db.get_table("StepTimeTable")]
    assert len(rows) == n == len(recs)
    for ph, name in names.items():
        ref_us = np.array([list(r["events"][name].values())[0]["duration_ms"] * 1000.0 for r in rows])
        mine_us = recs["dur_ns"][:, ph].astype(np.float64) / 1000.0
        assert all(list(r["events"][name].values())[0]["is_gpu"] for r in rows)
        tol = 2.0 + 0.01 * mine_us
        assert (ref_us <= mine_us + tol).all(), (name, float((ref_us - mine_us).max()))
        # the reference's pair sits inside ours: the gap is two event records + launch gaps
        assert np.median(mine_us - ref_us) < 25.0, float(np.median(mine_us - ref_us))
        assert abs(mine_us.mean() - ref_us.mean()) <= 0.005 * ref_us.mean() + 25.0
    eng.close()
