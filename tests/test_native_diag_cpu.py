"""CPU: the host-side C++ rule engines of libtraceml_b200.so (tml_diag_*) against
the reference's golden diagnoses.  Inputs (rank means, series band means) are
derived with the oracle here; on the GPU they come from the reduce kernels
(tests/test_gpu_parity.py runs the same comparison end to end)."""
import ctypes as C

import numpy as np
import pytest

from oracle import step_memory_oracle, step_time_oracle
from helpers import (assert_struct, golden_cases, oracle_mem_rows, oracle_time_rows, plain,
                     proc_replay_for, step_replay_for, strip_device)
from traceml_b200 import _abi, sections
from traceml_b200.reduce import trend_layout

STEP = golden_cases("step")
PROC = golden_cases("process")


def _trend(series, lay):
    t = _abi.TrendIn()
    if series is None or lay is None:
        t.valid = 0
        return t
    a = np.asarray(series, dtype=np.float64)
    t.valid = 1
    t.baseline_avg = float(a[lay[0][0]:lay[0][1]].sum() / (lay[0][1] - lay[0][0]))
    t.mid_avg = float(a[lay[1][0]:lay[1][1]].sum() / (lay[1][1] - lay[1][0]))
    t.recent_avg = float(a[lay[2][0]:lay[2][1]].sum() / (lay[2][1] - lay[2][0]))
    return t


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_time_rules_native(g):
    recs = step_replay_for(g)
    o = step_time_oracle.step_time_section(oracle_time_rows(recs, g["window"]), max_rows=g["window"])
    aligned = o["data"]["aligned_summary"]
    win = o["data"]["aligned_window"]
    din = _abi.StDiagIn()
    din.n_ranks, din.max_rows = len(aligned), g["window"]
    din.n_common = win["steps_analyzed"]
    din.completed_step = win["end_step"] or 0
    for i, (r, s) in enumerate(sorted(aligned.items())):
        rm = din.ranks[i]
        rm.rank, rm.steps_analyzed = r, s["steps_analyzed"]
        rm.dataloader_ms, rm.forward_ms = s["avg_dataloader_ms"], s["avg_forward_ms"]
        rm.backward_ms, rm.optimizer_ms = s["avg_backward_ms"], s["avg_optimizer_ms"]
        rm.step_cpu_ms = s["avg_step_cpu_ms"]
    if aligned and win["steps_analyzed"]:
        steps = step_time_oracle.common_suffix_steps(o["data"]["aligned_step_metrics"], g["window"])
        lay = trend_layout(len(steps), min_points=200, warmup_frac=0.10)
        which = "worst" if len(aligned) <= 1 else "median"
        ser = {k: step_time_oracle.metric_series(k, steps, o["data"]["aligned_step_metrics"])
               for k in ("step_time", "wait_proxy", "dataloader_fetch")}
        din.trend_step = _trend(ser["step_time"][which], lay)
        din.trend_wait = _trend(ser["wait_proxy"][which], lay)
        din.trend_dl = _trend(ser["dataloader_fetch"][which], lay)
    got = _abi.diag_json("tml_diag_step_time", din)
    assert_struct(plain(got), g["step_time"]["diagnosis"], "diagnosis")


@pytest.mark.parametrize("g", STEP, ids=[g["case"] for g in STEP])
def test_step_memory_rules_native(g):
    recs = step_replay_for(g)
    cases = [(None, g["step_memory"]["diagnosis"])]
    if "step_memory_with_total" in g:
        cases.append((g["step_memory_with_total"]["gpu_total_bytes"],
                      g["step_memory_with_total"]["diagnosis"]))
    win = step_memory_oracle.aligned_window(oracle_mem_rows(recs), g["window"])
    metrics = step_memory_oracle.combined_metrics(win)
    for total, ref in cases:
        din = _abi.MemDiagIn()
        n = len(win["steps"])
        din.steps_used, din.window_size = n, g["window"]
        din.completed_step = win["steps"][-1] if n else 0
        din.ranks_seen = win["global_ranks_seen"]
        din.gpu_total_bytes = float(total) if total else 0.0
        din.n_metrics = len(metrics)
        ranks = sorted(win["per_global_rank"])
        lay = trend_layout(n, min_points=50, warmup_frac=0.0)
        for mi, m in enumerate(metrics):
            mm = din.metric[mi]
            mm.n_ranks = len(ranks)
            for i, r in enumerate(ranks):
                mm.ranks[i] = r
                mm.rank_peak[i] = max(v[mi] for v in win["per_global_rank"][r].values())
            mm.trend_worst = _trend(m["series"]["worst"], lay)
            mm.trend_median = _trend(m["series"]["median"], lay)
            mm.points = n
            tws = min(n, 1000)
            mm.tail_first = m["series"]["worst"][n - tws]
            mm.tail_last = m["series"]["worst"][-1]
        got = strip_device(plain(_abi.diag_json("tml_diag_step_memory", din)))
        ref = strip_device(ref)
        assert_struct(got["primary"], ref["primary"], "primary")
        assert_struct(got["issues"], ref["issues"], "issues")
        for k, sig in ref["metric_attribution"].items():
            assert_struct({x: got["metric_attribution"][k][x] for x in sig}, sig, f"attr.{k}")


def _agg_from_records(recs, max_rows):
    r = recs[-max_rows:]
    a = _abi.ProcAgg()
    a.n = len(r)
    if not len(r):
        a.max_ratio = -1.0
        return a
    has = (r["flags"] & 2) != 0
    a.n_gpu = int(has.sum())
    a.ts_min, a.ts_max = float(r["ts"].min()), float(r["ts"].max())
    import math

    a.sum_cpu, a.max_cpu = math.fsum(r["cpu_pct"].tolist()), float(r["cpu_pct"].max())
    a.sum_cpu_lo = 0.0
    # byte sums are exact integers, as K6 gives them (Python ints: no u64 wrap in numpy's sum)
    a.sum_rss, a.max_rss = sum(int(x) for x in r["rss"]), float(r["rss"].max())
    if a.n_gpu:
        used = r["mem_alloc"][has].astype(np.float64)
        resv = r["mem_resv"][has].astype(np.float64)
        a.sum_used, a.max_used = sum(int(x) for x in r["mem_alloc"][has]), float(used.max())
        a.sum_resv, a.max_resv = sum(int(x) for x in r["mem_resv"][has]), float(resv.max())
        a.max_total = float(r["mem_total"][has].max())
        pos = used > 0
        a.max_ratio = float((resv[pos] / used[pos]).max()) if pos.any() else -1.0
    else:
        a.max_ratio = -1.0
    a.max_cores = int(r["cpu_cores"].max())
    a.any_gpu_available = int(((r["flags"] & 1) != 0).any())
    return a


@pytest.mark.parametrize("g", PROC, ids=[g["case"] for g in PROC])
def test_process_rules_native(g):
    import replay

    procs = proc_replay_for(g)
    aggs = {r: sections.proc_agg_dict(_agg_from_records(procs[r], g["max_rows"]),
                                      ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=g["ranks"])
            for r in procs}
    got = plain(sections.build_process(aggs))
    ref = g["process"]
    assert_struct(got["primary"], ref["diagnosis"]["primary"], "primary")
    assert_struct(got["issues"], ref["diagnosis"]["issues"], "issues")
    ragg = dict(ref["aggregate"])
    ragg.pop("gpu_mem_reserved_overhang_ratio", None)
    assert_struct(got["aggregate"], ragg, "aggregate")
    for r, pr in ref["per_global_rank"].items():
        mine = got["per_global_rank"][r]
        assert_struct(mine, {k: pr[k] for k in mine}, f"rank{r}")


def test_step_time_empty_is_null():
    din = _abi.StDiagIn()
    din.n_ranks = 0
    assert _abi.diag_json("tml_diag_step_time", din) is None
