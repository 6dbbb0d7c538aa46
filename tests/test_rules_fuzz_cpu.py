"""Seeded random scenarios: the host C++ rule engines + section objects (through the numpy
engine double, so no GPU) against the oracle -- beyond the committed golden cases."""
import random

import pytest
import torch

from helpers import (assert_struct, oracle_mem_rows, oracle_proc_rows, oracle_time_rows, plain,
                     strip_device)

STEP_SC = ["balanced", "input_straggler", "compute_straggler", "straggler", "input_bound", "wait_heavy",
           "compute_bound", "warmup", "ragged", "trend_worsening", "duplicates", "empty_rank", "no_overlap",
           "mem_creep_confirmed", "mem_creep_early", "mem_imbalance", "mem_pressure"]
PROC_SC = ["normal", "very_high_gpu", "high_gpu", "overhang", "imbalance", "high_rss", "high_cpu", "no_gpu"]


def _cases(n, seed):
    rng = random.Random(seed)
    return [(rng.choice(STEP_SC), rng.choice(PROC_SC), rng.choice([1, 2, 3, 4, 6, 8]),
             rng.choice([40, 90, 260, 520]), rng.randrange(10_000), rng.choice([1, 3, 29, 128, 10_000]))
            for _ in range(n)]


@pytest.mark.parametrize("scenario,pscenario,R,S,seed,W", _cases(40, 4242))
def test_sections_vs_oracle_random(scenario, pscenario, R, S, seed, W):
    from fake_engine import FakeEngine
    from oracle import process_oracle, step_memory_oracle, step_time_oracle
    import replay
    from traceml_b200 import sections

    recs = replay.make_step_replay(scenario, R, S, seed)
    cut = random.Random(seed)
    for r in recs:  # lagging ranks: with a tiny window the memory candidate limit (20 W) binds
        if cut.random() < 0.3 and len(recs[r]) > 3:
            recs[r] = recs[r][:cut.randrange(1, len(recs[r]))]
    procs = replay.make_proc_replay(pscenario, R, 150, seed)
    se = sections.SummaryEngine([FakeEngine(recs[r], procs[r], dense_ok=bool(seed & 1)) for r in range(R)],
                                ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)
    se.reducer.device = torch.device("cpu")
    got = se.build(W, W)
    red = got.pop("reduce")
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, W), max_rows=W)
    g = got["step_time"]
    assert_struct(plain(g["data"]), plain({k: o["data"][k] for k in g["data"]}), "time.data")
    assert_struct(plain(g["diagnosis"]), plain(o["diagnosis"]), "time.diagnosis")
    for k in ("average", "median", "worst"):
        assert_struct(plain(g["global"][k]), plain(o["global"][k]), f"time.global.{k}")
    assert_struct(plain(g["overview"]), plain(o["overview"]), "time.overview")
    mo = step_memory_oracle.step_memory_section(oracle_mem_rows(recs), window_size=W,
                                                gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
    gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
    assert_struct(gd["primary"], od["primary"], "mem.primary")
    assert_struct(gd["issues"], od["issues"], "mem.issues")
    assert_struct(plain(got["step_memory"]["per_global_rank"]), plain(mo["per_global_rank"]), "mem.rows")
    assert_struct(plain(got["step_memory"]["global"]), plain(mo["global"]), "mem.global")
    # the whole Process section: the rule engine on the same aggregates, one host's constants
    aggs = {r: dict(a, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R) for r, a in red.proc_aggs.items()}
    assert_struct(plain(got["process"]), plain(sections.build_process(aggs)), "process", rel=0.0)
    po = process_oracle.process_section(oracle_proc_rows(procs, R), max_rows=W)
    assert_struct(plain(got["process"]["primary"]), plain(po["diagnosis"]["primary"]), "proc.primary")
    assert_struct(plain(got["process"]["issues"]), plain(po["diagnosis"]["issues"]), "proc.issues")
