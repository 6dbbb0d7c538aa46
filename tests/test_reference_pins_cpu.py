"""CPU: the known-answer vectors the REFERENCE'S OWN TESTS hold for this path (SURVEY 8c),
restated here as data and run against (1) the oracle, (2) the native C++ rule engines of
libtraceml_b200.so (host code, no GPU), and -- where the reference is importable (build
container) -- (3) the kept payload builder fed with the native diagnosis, for the exact card
strings.  Each case names the reference test it restates (paths under the reference's tests/).

Two kinds of vectors exist in the reference's tests.  Rank-level ones (rank means in, diagnosis
out) fit the native engines as they are.  Metric-level ones set summary fields independently of
each other (a worst peak of 6 GiB next to ``skew_pct = 0``): the native engines DERIVE median,
worst and skew from per-rank values, so those vectors run on the oracle as written and on the
native engine through per-rank values chosen to realise the same signals."""
import math

import pytest

from oracle import process_oracle, step_memory_oracle, step_time_oracle, trend_oracle
from helpers import plain
from traceml_b200 import _abi
from traceml_b200.reduce import trend_layout

GIB = 1024.0 * 1024.0 * 1024.0


# ------------------------------------------------------------------------------ step time
def _rank(*, steps=64, dataloader=5.0, forward=30.0, backward=50.0, optimizer=10.0, step_cpu=None):
    """reporting/summary/test_step_time_card.py:24-47 -- the rank summary the card tests build."""
    compute = forward + backward + optimizer
    eff = max(step_cpu if step_cpu is not None else compute, compute)
    return {"steps_analyzed": steps, "avg_dataloader_ms": dataloader, "avg_forward_ms": forward,
            "avg_backward_ms": backward, "avg_optimizer_ms": optimizer, "avg_step_cpu_ms": eff,
            "avg_traced_step_ms": eff, "avg_gpu_compute_ms": compute,
            "avg_total_step_ms": dataloader + eff}


def _native_step_time(ranks, max_rows):
    din = _abi.StDiagIn()
    din.n_ranks, din.max_rows = len(ranks), max_rows
    din.n_common = min((s["steps_analyzed"] for s in ranks.values()), default=0)
    din.completed_step = 0
    for i, (r, s) in enumerate(sorted(ranks.items())):
        rm = din.ranks[i]
        rm.rank, rm.steps_analyzed = r, s["steps_analyzed"]
        rm.dataloader_ms, rm.forward_ms = s["avg_dataloader_ms"], s["avg_forward_ms"]
        rm.backward_ms, rm.optimizer_ms = s["avg_backward_ms"], s["avg_optimizer_ms"]
        rm.step_cpu_ms = s["avg_step_cpu_ms"]
    return plain(_abi.diag_json("tml_diag_step_time", din))


def _oracle_step_time(ranks, max_rows):
    return step_time_oracle.diagnose_summary(step_time_oracle.rank_signals_from_summary(ranks), max_rows=max_rows)


# (reference test, ranks, status, issue kinds that must be present, exact issue-kind set or None,
#  card lines the kept builder must print)
CARDS = [
    ("test_step_time_card.py:101-127 balanced",
     {0: _rank(dataloader=20.0, forward=20.0, backward=35.0, optimizer=5.0, step_cpu=70.0),
      1: _rank(dataloader=20.0, forward=21.0, backward=34.0, optimizer=5.0, step_cpu=70.0)},
     "BALANCED", set(), None, ["- Diagnosis: BALANCED", "- Why: No clear timing bottleneck."]),
    ("test_step_time_card.py:130-153 compute bound 90.0/97.0",
     {0: _rank(dataloader=2.0, forward=20.0, backward=65.0, optimizer=5.0, step_cpu=95.0)},
     "COMPUTE-BOUND", {"COMPUTE_BOUND"}, None,
     ["- Stats: total 97.0ms | input 2.0ms | compute 90.0ms",
      "- Why: Compute dominated (90.0ms/97.0ms); backward was largest."]),
    ("test_step_time_card.py:156-174 input bound 40.0/140.0",
     {0: _rank(dataloader=40.0, forward=20.0, backward=35.0, optimizer=5.0, step_cpu=100.0)},
     "INPUT-BOUND", {"INPUT_BOUND"}, None,
     ["- Why: Input loading took a large share (40.0ms/140.0ms)."]),
    ("test_step_time_card.py:177-195 wait heavy 30.0/102.0",
     {0: _rank(dataloader=2.0, forward=20.0, backward=45.0, optimizer=5.0, step_cpu=100.0)},
     "WAIT-HEAVY", {"WAIT_HEAVY"}, None,
     ["- Why: Wait was high inside the total step (30.0ms/102.0ms)."]),
    ("test_step_time_card.py:198-226 input straggler r1 70.0/40.0",
     {0: _rank(dataloader=10.0, forward=40.0, backward=130.0, step_cpu=219.0),
      1: _rank(dataloader=70.0, forward=40.0, backward=130.0, step_cpu=219.0)},
     "INPUT STRAGGLER", {"INPUT_STRAGGLER"}, {"INPUT_STRAGGLER"},
     ["- Why: r1 input was slower than median global rank (70.0/40.0ms)."]),
    ("test_step_time_card.py:229-247 compute straggler r1 260.0/220.0",
     {0: _rank(dataloader=10.0, forward=40.0, backward=130.0),
      1: _rank(dataloader=10.0, forward=90.0, backward=160.0)},
     "COMPUTE STRAGGLER", {"COMPUTE_STRAGGLER"}, {"COMPUTE_STRAGGLER"},
     ["- Why: r1 compute was slower than median global rank (260.0/220.0ms)."]),
    ("test_step_time_card.py:250-279 combined straggler keeps all rank issues",
     {0: _rank(dataloader=10.0, forward=40.0, backward=130.0),
      1: _rank(dataloader=80.0, forward=90.0, backward=160.0)},
     "STRAGGLER", {"STRAGGLER", "INPUT_STRAGGLER", "COMPUTE_STRAGGLER"}, None,
     ["- Why: Input and compute varied across ranks."]),
    ("test_step_time_card.py:282-299 straggler has priority over wait heavy",
     {0: _rank(dataloader=10.0, forward=40.0, backward=130.0, step_cpu=350.0),
      1: _rank(dataloader=80.0, forward=90.0, backward=160.0, step_cpu=350.0)},
     "STRAGGLER", {"WAIT_HEAVY"}, None, ["- Diagnosis: STRAGGLER"]),
]


@pytest.mark.parametrize("case", CARDS, ids=[c[0] for c in CARDS])
def test_step_time_card_vectors(case):
    _, ranks, status, present, exact, _ = case
    for name, diag in (("oracle", _oracle_step_time(ranks, 64)), ("native", _native_step_time(ranks, 64))):
        assert diag["primary"]["status"] == status, name
        kinds = {i["kind"] for i in diag["issues"]}
        assert kinds >= present, (name, kinds)
        if exact is not None:
            assert kinds == exact, (name, kinds)
    # the two agree on everything, not only on the pinned fields
    from helpers import assert_struct

    assert_struct(_native_step_time(ranks, 64), plain(_oracle_step_time(ranks, 64)), "diagnosis")


def _reference_importable():
    try:
        from traceml_b200 import reporting
    except Exception:
        return False
    return reporting.reference_available()


@pytest.mark.parametrize("case", CARDS, ids=[c[0] for c in CARDS])
def test_step_time_card_strings_through_the_kept_builder(case):
    """The card text is the KEPT builder's; what is checked is that the native diagnosis carries
    everything the builder needs to print the reference's exact lines."""
    if not _reference_importable():
        pytest.skip("the reference is not installed in oracle/_ref")
    from traceml.reporting.sections.step_time.builder import build_step_time_payload
    from traceml_b200 import reporting

    _, ranks, status, _, _, lines = case
    window = {"alignment": "common_steps",
              "steps_analyzed": min(s["steps_analyzed"] for s in ranks.values()),
              "start_step": None, "end_step": None, "window_size": 64,
              "global_ranks_used": len(ranks), "global_ranks_observed": len(ranks)}
    sec = {"data": {"training_steps": 100, "latest_step_observed": 99, "aligned_summary": ranks,
                    "aligned_window": window, "per_global_rank_summary": ranks, "max_rows": 64},
           "diagnosis": _native_step_time(ranks, 64)}
    data, diag = reporting.to_reference_step_time(sec, {})
    payload = build_step_time_payload(data, diag)
    assert payload["diagnosis"]["status"] == status
    for line in lines:
        assert line in payload["card"], (line, payload["card"])
    for banned in ("- Issues:", "- Note:", "- Global:", "- Dominant:"):  # _assert_compact_card
        assert banned not in payload["card"]


def test_step_time_no_data_is_null():
    """test_step_time_card.py:89-98: no ranks -> diagnosis None."""
    assert _oracle_step_time({}, 64) is None
    din = _abi.StDiagIn()
    din.n_ranks = 0
    assert _abi.diag_json("tml_diag_step_time", din) is None


def test_summary_policy_warmup_then_steps_used():
    """diagnostics/test_step_time.py:263-298: 40 steps -> WARMUP with the exact text; 60 -> steps_used 60."""
    r = {0: {"steps_analyzed": 40, "avg_dataloader_ms": 1.0, "avg_forward_ms": 20.0, "avg_backward_ms": 60.0,
             "avg_optimizer_ms": 10.0, "avg_step_cpu_ms": 100.0}}
    for diag in (_oracle_step_time(r, 100), _native_step_time(r, 100)):
        assert diag["primary"]["kind"] == "WARMUP"
        assert diag["primary"]["reason"] == "Only 40 steps per rank available; summary diagnosis requires 50."
    r[0]["steps_analyzed"] = 60
    for diag in (_oracle_step_time(r, 100), _native_step_time(r, 100)):
        assert diag["primary"]["steps_used"] == 60


def _time_metric(name, *, median, worst, worst_rank=1, skew=0.0, world_size=2, steps=64):
    """diagnostics/test_step_time.py:38-75 -- a metric with explicit summary fields."""
    return {"metric": name,
            "series": {"steps": list(range(steps)), "median": [median] * steps, "worst": [worst] * steps},
            "summary": {"window_size": steps, "steps_used": steps, "median_total": median,
                        "worst_total": worst, "worst_rank": worst_rank, "skew_ratio": skew, "skew_pct": skew},
            "coverage": {"expected_steps": steps, "steps_used": steps, "completed_step": steps,
                         "world_size": world_size, "ranks_present": world_size, "incomplete": False}}


def _single(step=100.0, dataloader=5.0, forward=30.0, backward=50.0, optimizer=10.0, wait=5.0):
    kw = dict(worst_rank=0, world_size=1)
    return [_time_metric("step_time", median=step, worst=step, **kw),
            _time_metric("dataloader_fetch", median=dataloader, worst=dataloader, **kw),
            _time_metric("forward", median=forward, worst=forward, **kw),
            _time_metric("backward", median=backward, worst=backward, **kw),
            _time_metric("optimizer_step", median=optimizer, worst=optimizer, **kw),
            _time_metric("wait_proxy", median=wait, worst=wait, **kw)]


# diagnostics/step_time/policy.py:16-35,49-53 -- the LIVE policy, which the reference's rule tests
# run under (``DEFAULT_THRESHOLDS``); the summary policy is the oracle's SUMMARY_THRESHOLDS
LIVE_THRESHOLDS = {
    "input_straggler_score_warn": 0.10, "input_straggler_score_crit": 0.20,
    "compute_straggler_score_warn": 0.10, "compute_straggler_score_crit": 0.20,
    "input_share_warn": 0.25, "input_share_crit": 0.35, "wait_share_warn": 0.15, "wait_share_crit": 0.25,
    "input_bound_max_skew": 0.06, "compute_bound_max_skew": 0.06,
    "compute_bound_share_warn": 0.85, "compute_bound_share_crit": 0.92, "min_steps_for_confident_diag": 20,
}
LIVE_MIN_STEPS_FOR_DIAG = 20


def _rule_kinds(metrics):
    ctx = step_time_oracle.build_context(metrics, dict(LIVE_THRESHOLDS), None)
    return {i["kind"] for i in step_time_oracle.run_rules(ctx)}


def test_metric_level_rule_vectors():
    """diagnostics/test_step_time.py:139-236: each rule with its trigger and its no-trigger input
    (live thresholds, as the reference test uses ``DEFAULT_THRESHOLDS``)."""
    inp = [_time_metric("step_time", median=220.0, worst=250.0),
           _time_metric("dataloader_fetch", median=10.0, worst=45.0, skew=0.2),
           _time_metric("forward", median=40.0, worst=40.0), _time_metric("backward", median=130.0, worst=130.0),
           _time_metric("optimizer_step", median=20.0, worst=20.0), _time_metric("wait_proxy", median=20.0, worst=20.0)]
    assert "INPUT_STRAGGLER" in _rule_kinds(inp)
    assert "INPUT_STRAGGLER" not in _rule_kinds(_single())
    comp = [_time_metric("step_time", median=240.0, worst=310.0),
            _time_metric("dataloader_fetch", median=10.0, worst=10.0),
            _time_metric("forward", median=40.0, worst=90.0, skew=0.2),
            _time_metric("backward", median=130.0, worst=160.0, skew=0.15),
            _time_metric("optimizer_step", median=20.0, worst=20.0), _time_metric("wait_proxy", median=40.0, worst=40.0)]
    assert "COMPUTE_STRAGGLER" in _rule_kinds(comp)
    assert "COMPUTE_STRAGGLER" not in _rule_kinds(_single())
    assert "INPUT_BOUND" in _rule_kinds(_single(step=100.0, dataloader=35.0, forward=20.0, backward=30.0,
                                                optimizer=5.0, wait=10.0))
    assert "INPUT_BOUND" not in _rule_kinds(_single(dataloader=10.0))
    assert "WAIT_HEAVY" in _rule_kinds(_single(wait=20.0))
    assert "WAIT_HEAVY" not in _rule_kinds(_single(wait=5.0))
    assert "COMPUTE_BOUND" in _rule_kinds(_single(dataloader=2.0, wait=3.0))
    assert "COMPUTE_BOUND" not in _rule_kinds(_single(dataloader=35.0, wait=3.0))


def test_metric_level_primary_combines_stragglers():
    """diagnostics/test_step_time.py:239-259."""
    m = [_time_metric("step_time", median=240.0, worst=330.0),
         _time_metric("dataloader_fetch", median=10.0, worst=45.0, skew=0.2),
         _time_metric("forward", median=40.0, worst=90.0, skew=0.2),
         _time_metric("backward", median=130.0, worst=160.0, skew=0.15),
         _time_metric("optimizer_step", median=20.0, worst=20.0), _time_metric("wait_proxy", median=40.0, worst=40.0)]
    res = step_time_oracle.diagnosis_result(m, dict(LIVE_THRESHOLDS))
    assert res["primary"]["kind"] == "STRAGGLER"
    assert {i["kind"] for i in res["issues"]} >= {"INPUT_STRAGGLER", "COMPUTE_STRAGGLER", "STRAGGLER"}


def test_policies_are_distinct():
    """diagnostics/test_step_time.py:262-276: the summary policy waits longer and tolerates more wait."""
    assert set(step_time_oracle.SUMMARY_THRESHOLDS) == set(LIVE_THRESHOLDS)
    assert step_time_oracle.SUMMARY_THRESHOLDS["wait_share_warn"] > LIVE_THRESHOLDS["wait_share_warn"]
    assert step_time_oracle.SUMMARY_MIN_STEPS_FOR_DIAG > LIVE_MIN_STEPS_FOR_DIAG


# ------------------------------------------------------------------------------ fixtures (sections)
def _events(dl, fwd, bwd, opt, step):
    return {f"_traceml_internal:{n}": {"cpu": {"is_gpu": False, "duration_ms": v, "n_calls": 1}}
            for n, v in (("dataloader_next", dl), ("forward_time", fwd), ("backward_time", bwd),
                         ("optimizer_step", opt), ("step_time", step))}


def test_single_rank_fixture_median_total_11():
    """reporting/summary/test_fixtures.py:586-656: 1 rank, steps 1..4, dl 1 / fwd 2 / bwd 3 / opt 1 /
    step 10, max_rows 4 -> median total 11.0; memory window of 4 steps (alloc 100 + step)."""
    rows = {0: [{"step": s, "events": _events(1.0, 2.0, 3.0, 1.0, 10.0)} for s in range(1, 5)]}
    o = step_time_oracle.step_time_section(rows, max_rows=4)
    assert o["global"]["median"]["total_step_ms"]["value"] == 11.0
    mem = {0: [(s, 100.0 + s, 200.0 + s) for s in range(1, 5)]}
    m = step_memory_oracle.step_memory_section(mem, window_size=4)
    assert len(m["window"]["steps"]) == 4 and m["window"]["global_ranks_used"] == 1
    sec = _sections_from_records({0: _records(range(1, 5), 1.0, 2.0, 3.0, 1.0, 10.0, 101.0, 201.0)}, 4)
    assert sec["step_time"]["global"]["median"]["total_step_ms"]["value"] == 11.0
    assert sec["step_memory"]["window"]["n_steps"] == 4


def _records(steps, dl, fwd, bwd, opt, wall, alloc0, resv0):
    """StepRecords (the ring's layout) of constant phases; peaks alloc0 + i, resv0 + i."""
    import numpy as np
    from traceml_b200.records import (FLAG_HAS_MEM, PHASE_BACKWARD, PHASE_DATALOADER, PHASE_FORWARD,
                                      PHASE_OPTIMIZER, PHASE_STEP, STEP_RECORD_DTYPE)

    steps = list(steps)
    rec = np.zeros(len(steps), dtype=STEP_RECORD_DTYPE)
    rec["step"] = steps
    for ph, ms in ((PHASE_DATALOADER, dl), (PHASE_FORWARD, fwd), (PHASE_BACKWARD, bwd), (PHASE_OPTIMIZER, opt),
                   (PHASE_STEP, wall)):
        rec["dur_ns"][:, ph] = int(round(ms * 1.0e6))
    rec["n_calls"][:] = 1
    rec["peak_alloc"] = [int(alloc0 + i) for i in range(len(steps))]
    rec["peak_resv"] = [int(resv0 + i) for i in range(len(steps))]
    rec["flags"] = FLAG_HAS_MEM
    rec["seq"] = np.arange(len(steps), dtype=np.uint64)
    return rec


def _sections_from_records(recs_by_rank, window):
    """The product's host code on CPU: the Python reduce driver over fake engines (numpy stand-ins
    for the kernels), then its output through the native section emitter."""
    import torch
    from fake_engine import FakeEngine
    from traceml_b200 import sections

    engines = [FakeEngine(recs_by_rank[r], None) for r in sorted(recs_by_rank)]
    se = sections.SummaryEngine(engines, ram_total=1.0e9, gpu_count=len(engines))
    se.reducer.device = torch.device("cpu")
    res = se.build(window, window)
    return plain({k: res[k] for k in ("step_time", "step_memory")})


def test_two_rank_fixture_aligned_window_5():
    """reporting/summary/test_fixtures.py:659-746: 2 ranks, steps 1..5, fwd 2 + rank, bwd 3 + rank,
    step 10 + rank, window 5 -> 5 aligned steps; memory: both ranks used, median idx among the ranks."""
    rows = {r: [{"step": s, "events": _events(1.0, 2.0 + r, 3.0 + r, 1.0, 10.0 + r)} for s in range(1, 6)]
            for r in (0, 1)}
    o = step_time_oracle.step_time_section(rows, max_rows=5)
    assert o["data"]["aligned_window"]["steps_analyzed"] == 5
    assert o["data"]["aligned_window"]["window_size"] == 5
    assert set(o["data"]["aligned_summary"]) == {0, 1}
    mem = {r: [(s, 100.0 + r * 20.0 + s, 200.0 + r * 30.0 + s) for s in range(1, 6)] for r in (0, 1)}
    m = step_memory_oracle.step_memory_section(mem, window_size=5)
    assert len(m["window"]["steps"]) == 5 and m["window"]["global_ranks_used"] == 2
    assert set(m["per_global_rank"]) == {"0", "1"}
    assert m["global"]["median"]["peak_allocated_bytes"]["idx"] in {"0", "1"}
    assert m["global"]["median"]["peak_reserved_bytes"]["idx"] in {"0", "1"}
    sec = _sections_from_records({r: _records(range(1, 6), 1.0, 2.0 + r, 3.0 + r, 1.0, 10.0 + r,
                                              101.0 + r * 20.0, 201.0 + r * 30.0) for r in (0, 1)}, 5)
    w = sec["step_time"]["data"]["aligned_window"]
    assert (w["steps_analyzed"], w["window_size"], w["global_ranks_used"]) == (5, 5, 2)
    assert sec["step_memory"]["window"]["n_steps"] == 5
    assert sec["step_memory"]["window"]["global_ranks_used"] == 2
    assert sec["step_memory"]["global"]["median"]["peak_allocated_bytes"]["idx"] in {"0", "1"}


# ------------------------------------------------------------------------------ step memory
def _mem_metric(*, worst_peak=90.0, median_peak=80.0, steps_used=60, skew_pct=0.0, worst_rank=1, ranks=2):
    """diagnostics/test_step_memory.py:65-98."""
    return {"metric": "peak_reserved", "device": "cuda:0",
            "series": {"steps": list(range(steps_used)), "median": [median_peak] * steps_used,
                       "worst": [worst_peak] * steps_used},
            "summary": {"window_size": steps_used, "steps_used": steps_used, "median_peak": median_peak,
                        "worst_peak": worst_peak, "worst_rank": worst_rank, "skew_ratio": skew_pct,
                        "skew_pct": skew_pct},
            "coverage": {"expected_steps": steps_used, "steps_used": steps_used, "completed_step": steps_used,
                         "world_size": ranks, "ranks_present": ranks, "incomplete": False}}


def _rising(*, steps_used=60, start=4.0 * GIB, end=6.0 * GIB, median_scale=0.5, skew_pct=0.0, worst_rank=1,
            ranks=2):
    """diagnostics/test_step_memory.py:101-141."""
    worst = [start + (end - start) * (i / float(steps_used - 1)) for i in range(steps_used)]
    median = [v * median_scale for v in worst]
    m = _mem_metric(worst_peak=max(worst), median_peak=max(median), steps_used=steps_used, skew_pct=skew_pct,
                    worst_rank=worst_rank, ranks=ranks)
    m["series"]["worst"], m["series"]["median"] = worst, median
    return m


def _native_mem(rank_series, gpu_total, window=None):
    """``rank_series[rank] = per-step peak_reserved``: the per-rank values the kernels would reduce.
    Band means / growth tail are taken exactly as K4b does (reduce.py:trend_layout)."""
    ranks = sorted(rank_series)
    n = len(rank_series[ranks[0]]) if ranks else 0
    din = _abi.MemDiagIn()
    din.steps_used, din.window_size = n, window or n
    din.completed_step = n
    din.ranks_seen = len(ranks)
    din.gpu_total_bytes = float(gpu_total) if gpu_total else 0.0
    din.n_metrics = 2 if n else 0
    lay = trend_layout(n, min_points=50, warmup_frac=0.0)

    def band(series):
        t = _abi.TrendIn()
        if lay is None:
            t.valid = 0
            return t
        t.valid = 1
        for name, (lo, hi) in zip(("baseline_avg", "mid_avg", "recent_avg"), lay):
            setattr(t, name, float(sum(series[lo:hi]) / (hi - lo)))
        return t

    for mi in range(din.n_metrics):
        mm = din.metric[mi]
        mm.n_ranks = len(ranks)
        cols = list(zip(*[rank_series[r] for r in ranks]))
        worst = [max(c) for c in cols]
        med = [step_memory_oracle.median2(c) for c in cols]
        for i, r in enumerate(ranks):
            mm.ranks[i] = r
            mm.rank_peak[i] = max(rank_series[r])
        mm.trend_worst, mm.trend_median = band(worst), band(med)
        mm.points = n
        tws = min(n, 1000)
        mm.tail_first, mm.tail_last = worst[n - tws], worst[-1]
    return plain(_abi.diag_json("tml_diag_step_memory", din))


def _kinds(diag):
    return [i["kind"] for i in diag["issues"] if i["metric"] == "peak_reserved"]


def test_memory_primary_high_pressure():
    """diagnostics/test_step_memory.py:186-193: worst 96 / median 80 of 100 bytes -> HIGH_PRESSURE first."""
    o = step_memory_oracle.diagnose_summary([_mem_metric(worst_peak=96.0, median_peak=80.0)], gpu_total_bytes=100.0)
    assert o["primary"]["kind"] == "HIGH_PRESSURE" and o["issues"][0]["kind"] == "HIGH_PRESSURE"
    n = _native_mem({0: [64.0] * 60, 1: [96.0] * 60}, 100.0)   # median (64 + 96) / 2 = 80
    assert n["primary"]["kind"] == "HIGH_PRESSURE" and n["issues"][0]["kind"] == "HIGH_PRESSURE"


def test_memory_rule_priority_pressure_imbalance_creep():
    """diagnostics/test_step_memory.py:196-208: 4 -> 6 GiB ramp, skew 0.4, capacity 6.1 GiB ->
    [HIGH_PRESSURE, IMBALANCE, CREEP_CONFIRMED]."""
    o = step_memory_oracle.diagnose_summary([_rising(skew_pct=0.4)], gpu_total_bytes=6.1 * GIB)
    assert o["primary"]["kind"] == "HIGH_PRESSURE"
    assert [i["kind"] for i in o["issues"]] == ["HIGH_PRESSURE", "IMBALANCE", "CREEP_CONFIRMED"]
    worst = _rising()["series"]["worst"]
    # rank 1 = the ramp, rank 0 = (2 / 1.4 - 1) of it: median peak 6 / 1.4 GiB, skew 0.4, same growth
    n = _native_mem({0: [v * (2.0 / 1.4 - 1.0) for v in worst], 1: worst}, 6.1 * GIB)
    assert n["primary"]["kind"] == "HIGH_PRESSURE"
    assert _kinds(n) == ["HIGH_PRESSURE", "IMBALANCE", "CREEP_CONFIRMED"]
    assert math.isclose(n["metric_attribution"]["peak_reserved"]["skew_pct"], 0.4, rel_tol=1e-12)


def test_memory_primary_for_each_non_pressure_issue():
    """diagnostics/test_step_memory.py:211-252."""
    o = step_memory_oracle.diagnose_summary(
        [_mem_metric(worst_peak=100.0, median_peak=70.0, skew_pct=0.3)], gpu_total_bytes=1000.0)
    assert o["primary"]["kind"] == "IMBALANCE"
    assert _native_mem({0: [40.0] * 60, 1: [100.0] * 60}, 1000.0)["primary"]["kind"] == "IMBALANCE"

    o = step_memory_oracle.diagnose_summary([_rising()], gpu_total_bytes=100.0 * GIB)
    assert o["primary"]["kind"] == "CREEP_CONFIRMED"
    ramp = _rising()["series"]["worst"]
    n = _native_mem({0: ramp, 1: ramp}, 100.0 * GIB)           # identical ranks: skew 0, as the vector states
    assert n["primary"]["kind"] == "CREEP_CONFIRMED" and _kinds(n) == ["CREEP_CONFIRMED"]

    o = step_memory_oracle.diagnose_summary([_rising(end=4.1 * GIB)], gpu_total_bytes=100.0 * GIB)
    assert o["primary"]["kind"] == "CREEP_EARLY"
    ramp = _rising(end=4.1 * GIB)["series"]["worst"]
    n = _native_mem({0: ramp, 1: ramp}, 100.0 * GIB)
    assert n["primary"]["kind"] == "CREEP_EARLY" and n["primary"]["status"] == "MEMORY RISING"

    o = step_memory_oracle.diagnose_summary([_mem_metric(worst_peak=90.0, median_peak=88.0)], gpu_total_bytes=1000.0)
    assert o["primary"]["kind"] == "BALANCED"
    assert _native_mem({0: [86.0] * 60, 1: [90.0] * 60}, 1000.0)["primary"]["kind"] == "BALANCED"

    assert step_memory_oracle.diagnose_summary([])["primary"]["kind"] == "NO_DATA"
    assert _native_mem({}, None)["primary"]["kind"] == "NO_DATA"


def test_memory_fifty_step_window_vectors():
    """diagnostics/test_step_memory_package.py:111-143: 49 steps -> "Need at least 50 completed
    steps."; 50 steps 4 -> 4.1 GiB -> MEMORY RISING with the exact reason; 4 -> 7.4 GiB -> creep."""
    def single(steps, start, end):
        return [start + (end - start) * (i / float(steps - 1)) for i in range(steps)]

    flat49 = _mem_metric(worst_peak=100.0, median_peak=90.0, steps_used=49, worst_rank=0, ranks=1)
    for d in (step_memory_oracle.diagnose_summary([flat49]), _native_mem({0: [100.0] * 49}, None)):
        assert d["primary"]["kind"] == "NO_DATA"
        assert d["primary"]["reason"] == "Need at least 50 completed steps."
    for end, kind, status, reason in (
            (4.1 * GIB, "CREEP_EARLY", "MEMORY RISING", "peak reserved is rising from early to recent steps."),
            (7.4 * GIB, "CREEP_CONFIRMED", "MEMORY CREEP", "peak reserved is rising across the window.")):
        m = _rising(steps_used=50, end=end, median_scale=1.0, worst_rank=0, ranks=1)
        o = step_memory_oracle.diagnose_summary([m])
        n = _native_mem({0: single(50, 4.0 * GIB, end)}, None)
        for d in (o, n):
            top = [i for i in d["issues"] if i["metric"] == "peak_reserved"][0]
            assert (top["kind"], top["status"], top["summary"]) == (kind, status, reason)


def test_memory_issue_sort_uses_domain_priority():
    """diagnostics/test_step_memory.py:255-290."""
    issues = [{"kind": "CREEP_CONFIRMED", "severity": "warn", "score": 100.0, "metric": None},
              {"kind": "HIGH_PRESSURE", "severity": "warn", "score": 0.93, "metric": None},
              {"kind": "IMBALANCE", "severity": "warn", "score": 0.4, "metric": None}]
    assert [i["kind"] for i in step_memory_oracle.sort_mem_issues(issues)] == \
        ["HIGH_PRESSURE", "IMBALANCE", "CREEP_CONFIRMED"]


def test_memory_alignment_vector_native_means():
    """reporting/summary/test_step_memory.py:206-298 -- aligned window (2, 3), means 115.0 / 215.0 --
    is pinned on the oracle in test_oracle_golden.py; here the same rows give the same per-rank
    window means whichever rank is asked."""
    rows = {0: [(1, 100.0, 200.0), (2, 110.0, 210.0), (3, 120.0, 220.0)],
            1: [(2, 111.0, 211.0), (3, 121.0, 221.0), (4, 131.0, 231.0)]}
    o = step_memory_oracle.step_memory_section(rows, window_size=2)
    assert o["per_global_rank"]["1"]["peak_allocated_bytes"] == 116.0
    assert o["per_global_rank"]["1"]["peak_reserved_bytes"] == 216.0


# ------------------------------------------------------------------------------ process
def _proc_data(per_rank=None, **over):
    """diagnostics/test_process.py:28-87 (``_input`` / ``_rank``) in the oracle's section format."""
    def rank(rss_peak=200.0, used_peak=200.0, reserved_peak=240.0, total=1000.0, overhang=None):
        return {"ram_peak_bytes": rss_peak, "gpu_mem_used_peak_bytes": used_peak,
                "gpu_mem_reserved_peak_bytes": reserved_peak, "gpu_mem_total_bytes": total,
                "gpu_mem_reserved_overhang_ratio": overhang}

    agg = dict(first_ts=0.0, last_ts=10.0, process_samples=10, distinct_global_ranks=1,
               cpu_avg_percent=120.0, cpu_peak_percent=200.0, cpu_logical_core_count=8,
               ram_avg_bytes=100.0, ram_peak_bytes=200.0, ram_total_bytes=1000.0, gpu_available=True,
               gpu_count=1, gpu_mem_used_avg_bytes=100.0, gpu_mem_used_peak_bytes=200.0,
               gpu_mem_reserved_avg_bytes=120.0, gpu_mem_reserved_peak_bytes=240.0, gpu_mem_total_bytes=1000.0)
    agg.update(over)
    pr = {r: rank(**kw) for r, kw in (per_rank or {0: {}}).items()}
    return {"aggregate": agg, "per_global_rank": pr}


PROC_CASES = [
    ("very high gpu memory", dict(gpu_mem_reserved_peak_bytes=930.0), None, "VERY_HIGH_PROCESS_GPU_MEMORY"),
    ("high gpu memory", dict(gpu_mem_reserved_peak_bytes=850.0), None, "HIGH_PROCESS_GPU_MEMORY"),
    ("reserved overhang", dict(gpu_mem_used_peak_bytes=400.0, gpu_mem_reserved_peak_bytes=700.0),
     {0: dict(used_peak=400.0, reserved_peak=700.0)}, "GPU_MEMORY_RESERVED_OVERHANG"),
    ("rank imbalance", {}, {0: dict(used_peak=900.0, reserved_peak=900.0),
                            1: dict(used_peak=400.0, reserved_peak=400.0)}, "RANK_GPU_MEMORY_IMBALANCE"),
    ("high rss", dict(ram_peak_bytes=850.0), None, "HIGH_PROCESS_RSS"),
    ("high cpu", dict(cpu_avg_percent=700.0), None, "HIGH_PROCESS_CPU"),
]


@pytest.mark.parametrize("case", PROC_CASES, ids=[c[0] for c in PROC_CASES])
def test_process_primary_for_each_issue(case):
    """diagnostics/test_process.py:90-221: each condition alone is the primary; the defaults trigger nothing."""
    _, over, per_rank, kind = case
    d = process_oracle.diagnose(_proc_data(per_rank, **over))
    assert d["primary"]["kind"] == kind
    assert kind in {i["kind"] for i in d["issues"]}
    assert process_oracle.diagnose(_proc_data())["issues"] == ()


def test_process_priority_when_everything_triggers():
    """diagnostics/test_process.py:224-252."""
    d = process_oracle.diagnose(_proc_data(
        {0: dict(used_peak=900.0, reserved_peak=1000.0, overhang=1000.0 / 900.0),
         1: dict(used_peak=400.0, reserved_peak=700.0, overhang=700.0 / 400.0)},
        cpu_avg_percent=700.0, ram_peak_bytes=850.0, gpu_mem_used_peak_bytes=400.0,
        gpu_mem_reserved_peak_bytes=1000.0))
    assert d["primary"]["kind"] == "VERY_HIGH_PROCESS_GPU_MEMORY"
    assert [i["kind"] for i in d["issues"]] == [
        "VERY_HIGH_PROCESS_GPU_MEMORY", "GPU_MEMORY_RESERVED_OVERHANG", "RANK_GPU_MEMORY_IMBALANCE",
        "HIGH_PROCESS_RSS", "HIGH_PROCESS_CPU"]


def _native_proc(ranks, ram_total=1000.0, gpu_count=1):
    """Per-rank aggregates as K6 produces them (``tml_proc_agg``): ``ranks[r]`` holds n samples of
    (cpu, rss, used, reserved, total) constants plus explicit peaks."""
    aggs = {}
    for r, v in ranks.items():
        a = _abi.ProcAgg()
        n = v.get("n", 10)
        a.n = n
        a.n_gpu = n if v.get("gpu", True) else 0
        a.ts_min, a.ts_max = 0.0, 10.0
        a.sum_cpu, a.max_cpu, a.sum_cpu_lo = v.get("cpu_avg", 120.0) * n, v.get("cpu_peak", 200.0), 0.0
        # byte sums are exact integers (u64), as K6 gives them
        a.sum_rss, a.max_rss = int(v.get("rss_avg", 100) * n), v.get("rss_peak", 200.0)
        if a.n_gpu:
            a.sum_used, a.max_used = int(v.get("used_avg", 100) * n), v.get("used_peak", 200.0)
            a.sum_resv, a.max_resv = int(v.get("resv_avg", 120) * n), v.get("resv_peak", 240.0)
            a.max_total = v.get("total", 1000.0)
            a.max_ratio = v.get("overhang", a.max_resv / a.max_used)
        else:
            a.max_ratio = -1.0
        a.max_cores = 8
        a.any_gpu_available = 1 if v.get("gpu", True) else 0
        from traceml_b200 import sections

        aggs[r] = sections.proc_agg_dict(a, ram_total=ram_total, gpu_count=gpu_count if v.get("gpu", True) else 0)
    from traceml_b200 import sections

    return plain(sections.build_process(aggs))


def test_process_vectors_on_the_native_engine():
    """The same conditions through ``tml_diag_process`` (per-rank aggregates in, as the reduce
    kernel hands them over).  The aggregate is DERIVED from the ranks there, so a vector that sets
    a rank's reserved peak to 930 of 1000 bytes also has a 4.65x overhang: the primary is what the
    reference's priority list says, the other issues ride along."""
    assert _native_proc({0: {}})["primary"]["kind"] == "NORMAL"
    assert _native_proc({0: dict(resv_peak=930.0)})["primary"]["kind"] == "VERY_HIGH_PROCESS_GPU_MEMORY"
    assert _native_proc({0: dict(resv_peak=850.0)})["primary"]["kind"] == "HIGH_PROCESS_GPU_MEMORY"
    d = _native_proc({0: dict(used_peak=400.0, resv_peak=700.0)})
    assert d["primary"]["kind"] == "GPU_MEMORY_RESERVED_OVERHANG"
    assert _native_proc({0: dict(rss_peak=850.0)})["primary"]["kind"] == "HIGH_PROCESS_RSS"
    assert _native_proc({0: dict(cpu_avg=700.0, cpu_peak=800.0)})["primary"]["kind"] == "HIGH_PROCESS_CPU"
    # test_process.py:255-270: the overhang is the rank-local peak ratio, reported for that rank
    d = _native_proc({0: dict(used_peak=1000.0, resv_peak=1200.0, total=2000.0, overhang=1.2),
                      1: dict(used_peak=100.0, resv_peak=180.0, total=2000.0, overhang=1.8)}, gpu_count=2)
    top = d["issues"][0]
    assert top["kind"] == "GPU_MEMORY_RESERVED_OVERHANG" and list(top["ranks"]) == [1]
    assert top["evidence"]["gpu_mem_reserved_overhang_ratio"] == 1.8
    # test_process.py:273-289: CPU-only run -> NORMAL without GPU wording
    d = _native_proc({0: dict(gpu=False)}, gpu_count=0)
    assert d["primary"]["kind"] == "NORMAL" and "GPU" not in d["primary"]["reason"] and d["issues"] == []
    # test_process.py:292-296: no samples -> NO_DATA, no rules run
    d = _native_proc({0: dict(n=0)})
    assert d["primary"]["kind"] == "NO_DATA" and d["issues"] == []


def test_process_overhang_uses_rank_local_ratio_oracle():
    """diagnostics/test_process.py:255-270 on the oracle."""
    d = process_oracle.diagnose(_proc_data(
        {0: dict(used_peak=1000.0, reserved_peak=1200.0, overhang=1.2),
         1: dict(used_peak=100.0, reserved_peak=180.0, overhang=1.8)},
        gpu_mem_used_peak_bytes=1000.0, gpu_mem_reserved_peak_bytes=1200.0, gpu_mem_total_bytes=2000.0))
    top = d["issues"][0]
    assert top["kind"] == "GPU_MEMORY_RESERVED_OVERHANG" and tuple(top["ranks"]) == (1,)
    assert top["evidence"]["gpu_mem_reserved_overhang_ratio"] == 1.8


# ------------------------------------------------------------------------------ trend core
def test_trend_core_vectors():
    """diagnostics/test_trend_core.py: rising series, history limit, short series."""
    ev = trend_oracle.trend_evidence([100.0 + float(i) for i in range(500)])
    assert ev["delta_vs_baseline"] > 0.0 and ev["delta_pct_vs_baseline"] is not None
    assert ev["recent_avg"] > ev["mid_avg"] > ev["baseline_avg"]
    ev = trend_oracle.trend_evidence([10.0] * 1000, history_limit=200, min_points=50)
    assert ev["truncated"] is True and ev["points_used"] == 200
    assert trend_oracle.trend_pct([1.0, 2.0, 3.0], min_points=50) is None
    # the band layout the kernels use (reduce.trend_layout) is the oracle's band arithmetic
    for n in (50, 199, 200, 500, 10_000, 12_345):
        lay = trend_layout(n, min_points=200, warmup_frac=0.10)
        series = [float(i * i % 97) for i in range(n)]
        ev = trend_oracle.trend_evidence(series)
        assert (lay is None) == (ev is None)
        if lay is not None:
            got = [sum(series[lo:hi]) / (hi - lo) for lo, hi in lay]   # global indices
            assert got == [ev["baseline_avg"], ev["mid_avg"], ev["recent_avg"]]
