"""tml_sections_json (csrc/tml_sections.cpp, host C++: no GPU needed) on every golden case, with
the Python reduce driver over engine doubles feeding it (the ``ReduceRunOut`` it fills): the section
objects must equal the reference's golden outputs, the oracle's rollups and, for the Process
section, the rule engine run directly on the same aggregates."""
import json
import os

import pytest
import torch

from helpers import (assert_struct, golden_cases, oracle_mem_rows, plain, proc_replay_for, step_replay_for,
                     strip_device)
from traceml_b200.sections import build_process

STEP = golden_cases("step")
PROC = golden_cases("process")


def build_sections(records, procs, window):
    """The sections of one build over engine doubles, and the per-rank process aggregates
    (with the host constants) they were built from."""
    from fake_engine import FakeEngine
    import replay
    from traceml_b200 import sections

    R = len(records) if records is not None else len(procs)
    empty = replay.make_step_replay("balanced", 1, 0, 0)[0]
    engines = [FakeEngine(records[r] if records is not None else empty,
                          procs[r] if procs is not None else None) for r in range(R)]
    se = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)
    se.reducer.device = torch.device("cpu")
    res = se.build(window, window)
    red = res.pop("reduce")
    aggs = {r: dict(a, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R) for r, a in red.proc_aggs.items()}
    return res, aggs


def _assert_step_memory_golden(got, ref):
    """The step-memory object against the reference's (as test_gpu_parity checks it on the GPU)."""
    assert got["training_steps"] == ref["training_steps"]
    assert got["latest_step_observed"] == ref["latest_step_observed"]
    assert_struct(plain(got["window"]), ref["window"], "golden.mem.window")
    assert_struct(plain(got["metrics"]), ref["metrics"], "golden.mem.metrics")
    assert_struct(plain(got["per_global_rank"]), ref["per_global_rank"], "golden.mem.rows")
    gd, rd = strip_device(plain(got["diagnosis"])), strip_device(ref["diagnosis"])
    assert_struct(gd["primary"], rd["primary"], "golden.mem.primary")
    assert_struct(gd["issues"], rd["issues"], "golden.mem.issues")
    for k, sig in rd["metric_attribution"].items():
        assert_struct({x: gd["metric_attribution"][k][x] for x in sig}, sig, f"golden.mem.attr.{k}")
    if ref["payload"].get("global") and ref["window"]["n_steps"]:
        for k in ("average", "median", "worst"):
            assert_struct(plain(got["global"][k]), ref["payload"]["global"][k], f"golden.mem.global.{k}")


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_native_sections_equal_python_sections(g):
    """The Python driver's reduce through the native emitter against the reference's own step-time
    and step-memory objects (data / diagnosis / rollups), with and without a GPU total."""
    import replay

    recs = step_replay_for(g)
    nat, _ = build_sections(recs, None, g["window"])
    assert_struct(plain(nat["step_time"]["data"]), g["step_time"]["data"], "golden.data")
    assert_struct(plain(nat["step_time"]["diagnosis"]), g["step_time"]["diagnosis"], "golden.diagnosis")
    for k in ("average", "median", "worst"):
        assert_struct(plain(nat["step_time"]["global"][k]), g["step_time"]["payload"]["global"][k], f"golden.global.{k}")
    assert isinstance(next(iter(nat["step_time"]["data"]["aligned_summary"]), 0), int)
    _assert_step_memory_golden(nat["step_memory"], g["step_memory"])
    if "step_memory_with_total" in g:  # process samples give the GPU total: the pressure rules
        procs = replay.make_proc_replay("normal", g["ranks"], 50, g["seed"])
        got = build_sections(recs, procs, g["window"])[0]["step_memory"]
        t = g["step_memory_with_total"]
        assert got["gpu_total_bytes"] == t["gpu_total_bytes"]
        gd, rd = strip_device(plain(got["diagnosis"])), strip_device(t["diagnosis"])
        assert_struct(gd["primary"], rd["primary"], "golden.pressure.primary")
        assert_struct(gd["issues"], rd["issues"], "golden.pressure.issues")


@pytest.mark.parametrize("g", PROC, ids=[g["case"] for g in PROC])
def test_native_process_section_equals_python(g):
    """The Process section: the rule engine run directly on the reduce's aggregates, and the
    reference's own diagnosis."""
    procs = proc_replay_for(g)
    nat, aggs = build_sections(None, procs, g["max_rows"])
    assert_struct(plain(nat["process"]), plain(build_process(aggs)), "process", rel=0.0)
    assert_struct(plain(nat["process"]["primary"]), g["process"]["diagnosis"]["primary"], "golden.primary")
    assert_struct(plain(nat["process"]["issues"]), g["process"]["diagnosis"]["issues"], "golden.issues")


@pytest.mark.parametrize("pattern", [(0, 0, 1, 1), (0, 0, 0, 0, 0, 0), (0, 1, 0, 1, 0), (1, 0), (0, 1, 2, 0, 1, 2, 0)])
def test_tie_breaks_with_identical_ranks(pattern):
    """Ranks holding identical records: every per-rank value ties, so median / worst ranks are
    decided purely by the tie-break rules (|delta|, value, rank / lowest rank wins) -- the
    native rollups must make the oracle's (the reference's) choices."""
    import replay
    from helpers import oracle_time_rows
    from oracle import step_memory_oracle, step_time_oracle

    base = replay.make_step_replay("input_straggler", 3, 260, seed=5)
    recs = {r: base[p].copy() for r, p in enumerate(pattern)}
    pbase = replay.make_proc_replay("imbalance", 3, 120, seed=5)
    procs = {r: pbase[p].copy() for r, p in enumerate(pattern)}
    nat, aggs = build_sections(recs, procs, 10_000)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, 10_000), max_rows=10_000)
    st = nat["step_time"]
    assert_struct(plain(st["data"]), plain({k: o["data"][k] for k in st["data"]}), "oracle.data")
    for k in ("average", "median", "worst"):
        assert_struct(plain(st["global"][k]), plain(o["global"][k]), f"oracle.global.{k}", rel=0.0)
    assert_struct(plain(st["overview"]), plain(o["overview"]), "oracle.overview", rel=0.0)
    assert_struct(plain(st["diagnosis"]), plain(o["diagnosis"]), "oracle.diagnosis", rel=0.0)
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=10_000)
    sm = nat["step_memory"]
    assert_struct(plain(sm["per_global_rank"]), plain(mo["per_global_rank"]), "oracle.mem.rows", rel=0.0)
    assert_struct(plain(sm["global"]), plain(step_memory_oracle.rollup_points(mo["per_global_rank"])),
                  "oracle.mem.global", rel=0.0)
    assert_struct(plain(nat["process"]), plain(build_process(aggs)), "process", rel=0.0)


def test_sections_json_of_reduce_results_from_several_threads():
    """The JSON strings of one call come from a per-thread bump arena (tml_internal.h) that is
    rewound when the outermost entry point returns: calls racing on different threads (ctypes
    drops the GIL) over the results of several builds must not see each other's memory."""
    import ctypes as C
    import threading

    from fake_engine import FakeEngine
    import replay
    from traceml_b200 import _abi, sections

    outs = {}
    for R in (1, 3, 8):
        W = 300
        recs = replay.make_step_replay("input_straggler", R, W, seed=R)
        procs = replay.make_proc_replay("normal", R, W, seed=R)
        se = sections.SummaryEngine([FakeEngine(recs[r], procs[r]) for r in range(R)],
                                    ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)
        se.reducer.device = torch.device("cpu")
        red = se.build(W, W).pop("reduce")
        outs[R] = (red.out, R, W)
    lib = _abi.lib()
    want = {}
    for R, (o, _, W) in outs.items():
        buf = C.create_string_buffer(1 << 18)
        args = _abi.SectionsArgs(float(replay.PROC_RAM_TOTAL_BYTES), R, W, W, 0)
        assert lib.tml_sections_json(C.byref(o), C.byref(args), buf, len(buf)) == 0
        want[R] = buf.value
    bad = []

    def worker(R):
        o, _, W = outs[R]
        buf = C.create_string_buffer(1 << 18)
        args = _abi.SectionsArgs(float(replay.PROC_RAM_TOTAL_BYTES), R, W, W, 0)
        for _ in range(300):
            if lib.tml_sections_json(C.byref(o), C.byref(args), buf, len(buf)) != 0 or buf.value != want[R]:
                bad.append(R)
                return

    threads = [threading.Thread(target=worker, args=(R,)) for R in (1, 3, 8, 1, 3, 8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not bad, bad


def test_sections_pickle_as_their_text():
    """A build's sections pickle (to hand them to another process) as their text and what the
    caller attached, unparsed or parsed and changed; the emitter's input does not travel."""
    import pickle

    import replay

    recs = replay.make_step_replay("input_straggler", 3, 120, seed=2)
    procs = replay.make_proc_replay("normal", 3, 60, seed=2)
    for parse_first in (False, True):
        res, _ = build_sections(recs, procs, 100)
        res["system"] = {"nodes": {}}
        if parse_first:
            res.pop("process")
        back = pickle.loads(pickle.dumps(res))
        assert back.raw == res.raw and back["system"] == {"nodes": {}}
        assert plain(back) == plain(res)
        assert ("process" in back) is not parse_first


def test_reduce_result_pickles_with_its_series():
    """The Python driver's reduce result travels with its sections: the result struct and the
    series it kept, so ``n_common``, ``exchange``, the series and every band field survive."""
    import pickle

    from fake_engine import FakeEngine
    import replay
    from traceml_b200 import sections

    recs = replay.make_step_replay("input_straggler", 3, 120, seed=2)
    procs = replay.make_proc_replay("normal", 3, 60, seed=2)
    se = sections.SummaryEngine([FakeEngine(recs[r], procs[r]) for r in range(3)],
                                ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=3)
    se.reducer.device = torch.device("cpu")
    res = se.build(100, 100)
    red = res["reduce"]
    back = pickle.loads(pickle.dumps(res))
    assert back.raw == res.raw
    got = back["reduce"]
    assert got.exchange == red.exchange == "local" and got.ranks == red.ranks == [0, 1, 2]
    assert got.proc_aggs == red.proc_aggs
    for kind in ("time", "mem"):
        a, b = getattr(red, kind), getattr(got, kind)
        assert b.n_common == a.n_common == 100 and b.shard == a.shard
        assert torch.equal(b.series, a.series)
        assert bytes(b.band_sum) == bytes(a.band_sum) and bytes(b.tail_last) == bytes(a.tail_last)
