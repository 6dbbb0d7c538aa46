"""CPU: the System section.  The oracle against the reference goldens (``==`` on floats), the
native rule engine (tml_diag_system) against the golden diagnoses, the shared sum arithmetic of
k_sys_reduce (csrc/tml_sys_sum.h) against CPython's sum(), and -- where the reference is
installed -- the whole final-summary envelope, System card included, against the reference's
FinalReportGenerator over the same rows."""
import ctypes as C
import glob
import json
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import system_cases as sc  # noqa: E402
from oracle import system_oracle  # noqa: E402

GOLDENS = [json.load(open(p)) for p in sorted(glob.glob(os.path.join(HERE, "golden", "system", "*.json")))
           if not p.endswith("INDEX.json")]
IDS = [g["case"] for g in GOLDENS]


def _rows(g):
    return [sc.wire_row(s) for s in sc.make_raw(g["case"])]


def _drop_gpu_idx(section):
    out = json.loads(json.dumps(section))
    for n in out["nodes"].values():
        n["per_gpu"] = {str(i): {k: v for k, v in q.items() if k != "gpu_idx"} for i, q in n["per_gpu"].items()}
    return out


def test_goldens_cover_every_issue_kind_and_geometry():
    kinds = {g["section"]["diagnosis"]["primary"]["kind"] for g in GOLDENS}
    issues = {i["kind"] for g in GOLDENS for i in g["section"]["diagnosis"]["issues"]}
    assert issues == set(system_oracle.SYSTEM_ISSUE_PRIORITY)
    assert {"NORMAL", "NO_DATA"} <= kinds
    assert {g["gpus"] for g in GOLDENS} >= {0, 1, 3, 4, 8, 16}
    assert any(g["samples"] == 1 for g in GOLDENS)
    assert any(g["window"] < g["samples"] for g in GOLDENS)


@pytest.mark.parametrize("g", GOLDENS, ids=IDS)
def test_oracle_equals_golden(g):
    from golden.make_system_golden import wire_digest

    rows = _rows(g)
    assert wire_digest(rows) == g["input_sha256"]
    mine = system_oracle.system_section(rows, g["identity"], g["window"])
    assert _drop_gpu_idx(mine) == json.loads(json.dumps(g["section"]))


@pytest.mark.parametrize("g", GOLDENS, ids=IDS)
def test_native_rules_equal_golden_diagnosis(g):
    from traceml_b200 import sections

    rows = _rows(g)
    sec = system_oracle.system_section(rows, g["identity"], g["window"])
    got = sections.build_system(sc.sys_agg_from_oracle(sec), g["identity"])
    want = g["section"]
    assert got["diagnosis"]["primary"] == want["diagnosis"]["primary"]
    assert [i["kind"] for i in got["diagnosis"]["issues"]] == [i["kind"] for i in want["diagnosis"]["issues"]]
    assert got["diagnosis"]["issues"] == want["diagnosis"]["issues"]
    assert _drop_gpu_idx(got) == json.loads(json.dumps(want))


# ----------------------------------------------------------------------------- shared sum header
def _host_sum(x, mode, nblk=1):
    from traceml_b200 import _abi

    a = np.ascontiguousarray(x, dtype=np.float64)
    out = C.c_double(0.0)
    _abi.check(_abi.lib().tml_sys_host_sum(a.ctypes.data if len(a) else None, len(a), mode, nblk, C.byref(out)),
               "tml_sys_host_sum")
    return out.value


def _families():
    rng = np.random.default_rng(20261016)
    yield "one_decimal", [round(float(v), 1) for v in rng.uniform(0, 100, 10_000)]
    yield "uniform_1e5", rng.uniform(0, 100, 100_000).tolist()  # Python floats: CPython's compensated sum
    yield "binades", (rng.uniform(0, 1, 10_000) * 2.0 ** rng.integers(-30, 30, 10_000)).tolist()
    yield "ties", [1.0] + [2.0 ** -53] * 10_001 + [3.0 * 2.0 ** -53]
    yield "ties_half", [2.0 ** 53, 1.0, 1.0, -0.0, 1.0] * 2_000
    yield "mixed_int_decimal", [float(rng.integers(0, 101)) if i % 3 else float(rng.uniform(0, 100)) / 7.0
                                for i in range(10_000)]
    yield "watts", [int(v) / 1000.0 for v in rng.integers(50_000, 700_001, 100_000)]
    yield "tiny_and_huge", [1e16, 1.0, -1e16, 3.0, 1e-300] * 2_000


@pytest.mark.parametrize("name,x", list(_families()), ids=[n for n, _ in _families()])
def test_cpython_restatement_equals_sum(name, x):
    assert _host_sum(x, 0) == sum(x)
    for k in (1, 2, 3, 5, 16):  # the per-sample loop runs over <= 16 GPUs
        assert _host_sum(x[:k], 0) == sum(x[:k])


@pytest.mark.parametrize("name,x", list(_families()), ids=[n for n, _ in _families()])
def test_double_double_window_sum_equals_sum(name, x):
    """The kernel's tree for several grid sizes.  CPython's compensated sum and a correctly
    rounded double-double agree unless the exact sum sits on a rounding boundary that the
    compensation itself rounds across; none of these families (ties included) does."""
    want = sum(x)
    for nblk in (1, 3, 40, 391):
        assert _host_sum(x, 1, nblk) == want, nblk


def test_double_double_matches_fsum_on_non_negative_streams():
    rng = np.random.default_rng(7)
    for n in (1, 31, 32, 33, 257, 10_001):
        x = rng.uniform(0, 100, n).tolist()
        assert _host_sum(x, 1, 5) == math.fsum(x) == sum(x)


# ----------------------------------------------------------------------------- whole envelope
class _SystemDouble:
    """Engine double carrying a system ring (the oracle's aggregates stand in for K6s)."""

    def __init__(self, inner, rows, identity):
        self._inner, self.rows, self.identity = inner, rows, identity
        self._rows_n = None

    def __getattr__(self, k):
        return getattr(self._inner, k)

    @property
    def sys_count(self):
        return len(self.rows)

    def sys_reduce_beside(self, max_rows, stream=0):
        self._rows_n = int(max_rows)

    def sys_reduce_collect(self):
        sec = system_oracle.system_section(self.rows, self.identity, self._rows_n)
        return sc.sys_agg_from_oracle(sec)


@pytest.mark.parametrize("case,scenario,pscenario,R,S,W", [
    ("several_issues_g8", "input_straggler", "normal", 4, 460, 10_000),
    ("window_smaller_g8", "balanced", "high_cpu", 1, 300, 128),
    ("cpu_only", "balanced", "normal", 2, 200, 10_000),
    ("no_data", "balanced", "normal", 1, 120, 10_000),
])
def test_whole_envelope_with_system_equals_the_reference_report(tmp_path, case, scenario, pscenario, R, S, W):
    from traceml_b200 import reporting, sections

    if not reporting.reference_available():
        pytest.skip("the reference is not installed in oracle/_ref")
    import torch
    from fake_engine import FakeEngine
    from helpers import assert_struct, plain
    from traceml.reporting.final import build_final_report_generator

    import make_golden as mg
    import make_system_golden as msg
    import replay

    recs = replay.make_step_replay(scenario, R, S, seed=5)
    procs = replay.make_proc_replay(pscenario, R, 200, seed=5)
    ident = dict(sc.IDENTITY, world_size=R, local_world_size=R)
    rows = [sc.wire_row(s) for s in sc.make_raw(case)]
    db = str(tmp_path / "telemetry")
    mg.build_db(db, step_records=recs, proc_records=procs)
    msg.build_db(db, rows, ident)
    ref = build_final_report_generator(summary_window_rows=W).generate(db)
    engines = [FakeEngine(recs[r], procs[r]) for r in range(R)]
    engines[0] = _SystemDouble(engines[0], rows, ident)
    se = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R, system_identity=ident)
    se.reducer.device = torch.device("cpu")
    res = se.build(W, W)
    ids = {r: {"global_rank": r, "local_rank": r, "node_rank": 0, "hostname": "b200-box",
               "local_world_size": R, "world_size": R} for r in range(R)}
    env = reporting.build_final_summary(res, ids)
    assert set(ref) <= set(env)
    for k in ("system", "process", "step_time", "step_memory"):
        assert_struct(plain(env[k]), plain(ref[k]), k, rel=1e-12)
    assert env["duration_s"] == ref["duration_s"]
    assert env["text"] == ref["text"]


def test_fallback_text_has_a_system_line(monkeypatch):
    from traceml_b200 import reporting, sections

    monkeypatch.setattr(reporting, "reference_available", lambda: False)
    g = next(g for g in GOLDENS if g["case"] == "high_cpu_g8")
    sec = system_oracle.system_section(_rows(g), g["identity"], g["window"])
    system = sections.build_system(sc.sys_agg_from_oracle(sec), g["identity"])
    st = {"primary": {"status": "BALANCED", "reason": "r"}}
    res = {"step_time": {"diagnosis": st}, "step_memory": {"diagnosis": st}, "process": st, "system": system}
    env = reporting.build_final_summary(res, {0: dict(g["identity"])})
    assert env["text"].splitlines()[-1] == "System: HIGH CPU -- " + g["section"]["diagnosis"]["primary"]["reason"]
    assert env["system"] is system
