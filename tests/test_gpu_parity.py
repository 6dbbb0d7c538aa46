"""GPU parity tests proper: the CUDA path, through the C-ABI, against
 (a) the committed golden vectors (the reference's own outputs) and
 (b) the oracle on the same seeded inputs.

Every case plays all R ranks on one GPU (one engine per rank); the cross-rank
kernels see exactly what they would see after an NVLink exchange.
Tolerances (SURVEY 8d): step ids / rank ids / labels / issue order exact,
floats rel <= 1e-9 (summation order only)."""
import numpy as np
import pytest
import torch

from helpers import (REL_TOL, assert_struct, golden_cases, oracle_mem_rows, oracle_proc_rows,
                     oracle_time_rows, plain, proc_replay_for, step_replay_for, strip_device)

pytestmark = pytest.mark.gpu

STEP = golden_cases("step")
PROC = golden_cases("process")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _summary(records, window, procs=None, ring_slots=None, ranks=None):
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    R = len(records) if records is not None else len(procs)
    engines = []
    for r in range(R):
        n = len(records[r]) if records is not None else 0
        e = Engine(device=0, rank=r, world=R, ring_slots=ring_slots or max(64, n + 8),
                   proc_slots=max(64, (len(procs[r]) if procs else 0) + 8))
        if records is not None and n:
            e.load_steps(records[r])
        if procs is not None:
            e.load_procs(procs[r])
        engines.append(e)
    torch.cuda.synchronize()
    try:
        return sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                      gpu_count=R).build(window, window)
    finally:
        for e in engines:
            e.close()


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_time_vs_golden(cuda, g):
    recs = step_replay_for(g)
    got = _summary(recs, g["window"])["step_time"]
    ref = g["step_time"]
    assert_struct(plain(got["data"]), ref["data"], "data")
    assert_struct(plain(got["diagnosis"]), ref["diagnosis"], "diagnosis")
    for k in ("average", "median", "worst"):
        assert_struct(plain(got["global"][k]), ref["payload"]["global"][k], f"global.{k}")


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_memory_vs_golden(cuda, g):
    recs = step_replay_for(g)
    got = _summary(recs, g["window"])["step_memory"]
    ref = g["step_memory"]
    assert got["training_steps"] == ref["training_steps"]
    assert got["latest_step_observed"] == ref["latest_step_observed"]
    assert_struct(plain(got["window"]), ref["window"], "window")
    assert_struct(plain(got["metrics"]), ref["metrics"], "metrics")
    assert_struct(plain(got["per_global_rank"]), ref["per_global_rank"], "rows")
    gd, rd = strip_device(plain(got["diagnosis"])), strip_device(ref["diagnosis"])
    assert_struct(gd["primary"], rd["primary"], "primary")
    assert_struct(gd["issues"], rd["issues"], "issues")
    for k, sig in rd["metric_attribution"].items():
        assert_struct({x: gd["metric_attribution"][k][x] for x in sig}, sig, f"attr.{k}")
    if ref["payload"].get("global") and ref["window"]["n_steps"]:
        for k in ("average", "median", "worst"):
            assert_struct(plain(got["global"][k]), ref["payload"]["global"][k], f"global.{k}")


@pytest.mark.parametrize("g", [g for g in STEP if "step_memory_with_total" in g],
                         ids=[g["case"] for g in STEP if "step_memory_with_total" in g])
def test_step_memory_pressure_vs_golden(cuda, g):
    import replay

    recs = step_replay_for(g)
    procs = replay.make_proc_replay("normal", g["ranks"], 50, g["seed"])
    got = _summary(recs, g["window"], procs=procs)["step_memory"]
    t = g["step_memory_with_total"]
    assert got["gpu_total_bytes"] == t["gpu_total_bytes"]
    gd, rd = strip_device(plain(got["diagnosis"])), strip_device(t["diagnosis"])
    assert_struct(gd["primary"], rd["primary"], "primary")
    assert_struct(gd["issues"], rd["issues"], "issues")


@pytest.mark.parametrize("g", PROC, ids=[g["case"] for g in PROC])
def test_process_vs_golden(cuda, g):
    procs = proc_replay_for(g)
    got = plain(_summary(None, g["max_rows"], procs=procs)["process"])
    ref = g["process"]
    assert_struct(got["primary"], ref["diagnosis"]["primary"], "primary")
    assert_struct(got["issues"], ref["diagnosis"]["issues"], "issues")
    ragg = dict(ref["aggregate"])
    ragg.pop("gpu_mem_reserved_overhang_ratio", None)
    assert_struct(got["aggregate"], ragg, "aggregate")
    for r, pr in ref["per_global_rank"].items():
        mine = got["per_global_rank"][r]
        assert_struct(mine, {k: pr[k] for k in mine}, f"rank{r}")


def test_series_vs_oracle(cuda):
    """Per-step cross-rank median / worst series, element by element."""
    from oracle import step_memory_oracle, step_time_oracle
    import replay

    R, S, W = 5, 777, 512
    recs = replay.make_step_replay("ragged", R, S, seed=42)
    out = _summary(recs, W)["reduce"]
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, W), max_rows=W)
    steps = step_time_oracle.common_suffix_steps(o["data"]["aligned_step_metrics"], W)
    assert out.time.n_common == len(steps)
    ser = out.time.series.cpu().numpy()
    for mi, key in enumerate(step_time_oracle.METRIC_KEYS):
        ref = step_time_oracle.metric_series(key, steps, o["data"]["aligned_step_metrics"])
        np.testing.assert_allclose(ser[2 * mi], ref["median"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(ser[2 * mi + 1], ref["worst"], rtol=1e-12, atol=0)
    win = step_memory_oracle.aligned_window(oracle_mem_rows(recs), W)
    mets = step_memory_oracle.combined_metrics(win)
    mser = out.mem.series.cpu().numpy()
    for mi, m in enumerate(mets):
        np.testing.assert_array_equal(mser[12 + 2 * mi], np.asarray(m["series"]["median"]))
        np.testing.assert_array_equal(mser[13 + 2 * mi], np.asarray(m["series"]["worst"]))


def test_ring_wrap_and_window(cuda):
    """Ring smaller than the history: only the retained rows count
    (the reference prunes to 1.5 x window rows, sqlite_writer.py:394-424)."""
    from oracle import step_time_oracle
    import replay

    R, S, slots, W = 3, 1000, 300, 200
    recs = replay.make_step_replay("balanced", R, S, seed=5)
    got = _summary(recs, W, ring_slots=slots)["step_time"]
    kept = {r: recs[r][-slots:] for r in recs}
    ref = step_time_oracle.step_time_section(oracle_time_rows(kept, W), max_rows=W)
    assert_struct(plain(got["data"]["aligned_summary"]), plain(ref["data"]["aligned_summary"]), "aligned")
    assert_struct(plain(got["data"]["aligned_window"]), plain(ref["data"]["aligned_window"]), "window")
    assert_struct(plain(got["diagnosis"]), plain(ref["diagnosis"]), "diagnosis")


def test_large_window_properties(cuda):
    """BASELINE-size window (W = 10^6, R = 8): size-independent properties --
    identical ranks => median == worst == the rank's own series; permuting the
    ranks leaves every series bit-identical."""
    import replay
    from traceml_b200 import _abi, sections
    from traceml_b200.engine import Engine
    from traceml_b200.reduce import WindowReducer

    R, S = 8, 1_000_000
    base = replay.make_step_replay("balanced", 1, S, seed=9)[0]
    engines = [Engine(device=0, rank=r, world=R, ring_slots=S) for r in range(R)]
    for e in engines:
        e.load_steps(base)
    torch.cuda.synchronize()
    out = WindowReducer(engines).reduce(S)
    assert out.time.n_common == S and out.fused_pass
    ser = out.time.series
    assert torch.equal(ser[8], ser[9])       # step_time median == worst
    assert torch.equal(ser[12], ser[13])     # peak_allocated median == worst
    wall = torch.from_numpy((base["dur_ns"][:, 5].astype(np.float64) / 1.0e6)).cuda()
    comp = torch.from_numpy(((base["dur_ns"][:, 2].astype(np.float64) / 1e6
                              + base["dur_ns"][:, 3].astype(np.float64) / 1e6)
                             + base["dur_ns"][:, 4].astype(np.float64) / 1e6)).cuda()
    assert torch.equal(ser[8], torch.maximum(wall, comp))
    for e in engines:
        e.close()


# ---------------------------------------------------------------------------- native sequencing
def _run_out_fields(o):
    """What both reduce drivers must fill alike in a ReduceRunOut, as plain values: ``n_ranks``,
    ``fused_pass``, ``infos`` (but the kernel time each rank reports), ``procs``, and all of
    ``time`` / ``mem`` but where the series live.  A separate pass per section writes only that
    section's series rows, so the band sums and tails of the other rows are undefined and left
    out.  NaNs compare equal."""
    import ctypes as C

    def val(x, skip=()):
        if isinstance(x, C.Structure):
            return {f: val(getattr(x, f)) for f, _ in x._fields_ if f not in skip}
        if isinstance(x, C.Array):
            return [val(v) for v in x]
        return "nan" if isinstance(x, float) and x != x else x

    got = {"n_ranks": o.n_ranks, "fused_pass": o.fused_pass, "infos": [val(i, ("kernel_ms",)) for i in o.infos],
           "procs": val(o.procs)}
    for name, rows in (("time", slice(0, 12)), ("mem", slice(12, 16))):
        k = val(getattr(o, name), ("series",))
        for f in ("band_sum", "tail_first", "tail_last"):
            k[f] = k[f][rows]
        got[name] = k
    return got


@pytest.mark.parametrize("scenario,S,W,slots", [
    ("balanced", 300, 10_000, None), ("wait_heavy", 300, 128, None), ("duplicates", 240, 10_000, None),
    ("trend_worsening", 600, 10_000, None), ("mem_creep_confirmed", 300, 100, None),
    ("cpu_only", 120, 10_000, None), ("balanced", 1000, 200, 300), ("warmup", 40, 10_000, None),
    # tiny window over a long ring: the memory candidate limit (20 W) binds -- dense and holey rings
    ("balanced", 700, 3, None), ("duplicates", 700, 3, None), ("ragged", 900, 7, None),
])
def test_native_driver_equals_python_driver(cuda, scenario, S, W, slots):
    """tml_reduce_run (csrc/tml_summary.cpp) against the Python staging of the same C-ABI
    stages, one rank: every section, and the result struct both fill, identical bit for bit."""
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    recs = replay.make_step_replay(scenario, 1, S, seed=31)[0]
    procs = replay.make_proc_replay("overhang", 1, 300, seed=31)[0]
    out, series, facts, fields = {}, {}, {}, {}
    for native in (True, False):
        e = Engine(device=0, rank=0, world=1, ring_slots=slots or max(64, S + 8), proc_slots=512)
        e.load_steps(recs)
        e.load_procs(procs)
        torch.cuda.synchronize()
        try:
            se = sections.SummaryEngine([e], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1, native=native)
            assert se.reducer._native_ok() == native
            out[native] = se.build(W, W)
            again = se.build(W, W)  # workspace reuse
            red = again.pop("reduce")
            first = dict(out[native]); first.pop("reduce")
            assert_struct(plain(first), plain(again), "repeatable", rel=0.0)
            # the series live in the engine's workspace: copy them out before it closes
            series[native] = (red.time.series.clone() if red.time.n_common else None,
                              red.mem.series.clone() if red.mem.n_common else None)
            facts[native] = (red.exchange, red.fused_pass, red.time.n_common, red.mem.n_common)
            fields[native] = _run_out_fields(red.out)
        finally:
            e.close()
    a, b = out[True], out[False]
    a.pop("reduce"), b.pop("reduce")
    assert_struct(plain(a), plain(b), "native == python", rel=0.0)
    assert facts[True] == facts[False] and facts[True][0] == "local"
    assert fields[True] == fields[False]
    if series[True][0] is not None:
        assert torch.equal(series[True][0][:12], series[False][0][:12])
    if series[True][1] is not None:
        assert torch.equal(series[True][1][12:], series[False][1][12:])


@pytest.mark.parametrize("name", ["single_rank", "single_rank_wait", "cpu_only_r1"])
def test_native_driver_vs_reference_golden(cuda, name):
    """The native driver against the reference's own outputs (one-rank goldens)."""
    from helpers import load_golden
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    g = load_golden(name)
    recs = step_replay_for(g)
    e = Engine(device=0, rank=0, world=1, ring_slots=max(64, len(recs[0]) + 8), proc_slots=64)
    e.load_steps(recs[0])
    torch.cuda.synchronize()
    try:
        se = sections.SummaryEngine([e], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1)
        assert se.reducer._native_ok()
        got = se.build(g["window"], g["window"])
    finally:
        e.close()
    ref = g["step_time"]
    assert_struct(plain(got["step_time"]["data"]), ref["data"], "data")
    assert_struct(plain(got["step_time"]["diagnosis"]), ref["diagnosis"], "diagnosis")
    mref = g["step_memory"]
    assert_struct(plain(got["step_memory"]["metrics"]), mref["metrics"], "mem.metrics")
    assert_struct(strip_device(plain(got["step_memory"]["diagnosis"]))["primary"],
                  strip_device(mref["diagnosis"])["primary"], "mem.primary")


@pytest.mark.parametrize("R,scenario", [(11, "ragged"), (16, "compute_straggler")])
def test_more_than_eight_ranks(cuda, R, scenario):
    """R > 8 takes the generic (local-array, insertion-sort) reduce kernel and, in the live
    tick, numpy's blocked pairwise order for the per-step sums: both against the oracles."""
    from oracle import live_oracle, step_memory_oracle, step_time_oracle
    from traceml_b200 import records as rec_mod
    import replay
    from traceml_b200.engine import Engine
    from traceml_b200.live import StepCombinedComputer

    S, W = 330, 256
    recs = replay.make_step_replay(scenario, R, S, seed=77)
    got = _summary(recs, W)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, W), max_rows=W)
    g = got["step_time"]
    assert_struct(plain(g["data"]), plain({k: o["data"][k] for k in g["data"]}), "data")
    assert_struct(plain(g["diagnosis"]), plain(o["diagnosis"]), "diagnosis")
    steps = step_time_oracle.common_suffix_steps(o["data"]["aligned_step_metrics"], W)
    ser = got["reduce"].time.series.cpu().numpy()
    for mi, key in enumerate(step_time_oracle.METRIC_KEYS):
        ref = step_time_oracle.metric_series(key, steps, o["data"]["aligned_step_metrics"])
        np.testing.assert_allclose(ser[2 * mi], ref["median"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(ser[2 * mi + 1], ref["worst"], rtol=1e-12, atol=0)
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=W,
                                                gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
    assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")
    assert_struct(strip_device(plain(got["step_memory"]["diagnosis"]))["primary"],
                  strip_device(plain(mo["diagnosis"]))["primary"], "mem.primary")
    # live tick on the same rings
    engines = []
    for r in range(R):
        e = Engine(device=0, rank=r, world=R, ring_slots=512, proc_slots=64)
        if len(recs[r]):
            e.load_steps(recs[r])
        engines.append(e)
    torch.cuda.synchronize()
    try:
        tick = StepCombinedComputer(engines, window_size=100).compute_cli()
    finally:
        for e in engines:
            e.close()
    rows = {r: [rec_mod.step_record_to_wire(x, device=f"cuda:{r}") for x in recs[r]] for r in recs}
    assert_struct(plain(tick), plain(live_oracle.live_step_time(rows, window=100)), "live", rel=REL_TOL)


def _fuzz_cases(n, seed):
    import random

    rng = random.Random(seed)
    sc = ["balanced", "input_straggler", "compute_straggler", "straggler", "input_bound", "wait_heavy",
          "compute_bound", "warmup", "ragged", "trend_worsening", "duplicates", "empty_rank", "no_overlap",
          "mem_creep_confirmed", "mem_creep_early", "mem_imbalance", "mem_pressure"]
    return [(rng.choice(sc), rng.choice([1, 2, 3, 4, 6, 8]), rng.choice([40, 90, 260, 520]),
             rng.randrange(10_000), rng.choice([29, 128, 10_000]), rng.choice([None, None, 96]))
            for _ in range(n)]


@pytest.mark.parametrize("scenario,R,S,seed,W,slots", _fuzz_cases(24, 991))
def test_random_scenarios_vs_oracle(cuda, scenario, R, S, seed, W, slots):
    """Seeded random scenario / rank count / window / ring size through the kernels, against the
    oracle: data, diagnosis, rollups, memory rows (ring smaller than the history included)."""
    from oracle import step_memory_oracle, step_time_oracle
    import replay

    recs = replay.make_step_replay(scenario, R, S, seed)
    got = _summary(recs, W, ring_slots=slots)
    kept = {r: (recs[r][-slots:] if slots else recs[r]) for r in recs}
    o = step_time_oracle.step_time_section(oracle_time_rows(kept, W), max_rows=W)
    g = got["step_time"]
    assert_struct(plain(g["data"]), plain({k: o["data"][k] for k in g["data"]}), "data")
    assert_struct(plain(g["diagnosis"]), plain(o["diagnosis"]), "diagnosis")
    for k in ("average", "median", "worst"):
        assert_struct(plain(g["global"][k]), plain(o["global"][k]), f"global.{k}")
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows(kept), window_size=W,
                                                gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
    gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
    assert_struct(gd["primary"], od["primary"], "mem.primary")
    assert_struct(gd["issues"], od["issues"], "mem.issues")
    assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")


@pytest.mark.parametrize("W,dup", [(1, False), (3, False), (3, True), (7, True)])
def test_memory_candidate_limit_with_a_lagging_rank(cuda, W, dup):
    """A tiny window over a long ring with one rank far behind: the reference only aligns the
    newest max(20 W, W + 1) distinct steps of each rank (step_memory/loader.py:215), so the
    memory section finds no common window while the time section (last W rows) is unaffected."""
    from oracle import step_memory_oracle, step_time_oracle
    import replay

    recs = replay.make_step_replay("duplicates" if dup else "balanced", 3, 700, seed=123)
    recs[1] = recs[1][:200]
    got = _summary(recs, W)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, W), max_rows=W)
    assert_struct(plain(got["step_time"]["data"]), plain({k: o["data"][k] for k in got["step_time"]["data"]}), "data")
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=W,
                                                gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
    gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
    assert od["primary"]["reason"] == "No step-memory data yet."
    assert_struct(gd["primary"], od["primary"], "mem.primary")
    assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")
    assert got["step_memory"]["window"]["n_steps"] == 0
