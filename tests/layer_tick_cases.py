"""Shared by the layer-time tick tests: seeded layer-ring records, a numpy restatement of the
reference's five layer-time rules, the reference's own computer fed from the same records, and the
result comparison.

The five rules (renderers/layer_combined_time/compute.py):
  1. safe step: min over ranks that have both tables of min(last forward row's step, last backward
     row's step) (:111-135, :334-342);
  2. a layer is in a row when its ``*_calls > 0`` (LayerProfile.wire_rows);
  3. window / current: rows after the newest row with step < safe step; current = the newest of
     them whose step == safe step; none: the rank is missing in that direction (:156-168, :200-215);
  4. current = max over ranks, peak = max over the windows of the ranks with a current row (:170-187);
  5. worst rank: first maximum of fwd + bwd over ranks with a forward value, then the ranks with
     only a backward one (:239-253).
"""
from __future__ import annotations

import os
import sys
import types
from typing import Any, Dict, List

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.path.join(ROOT, "oracle", "_ref")


def layer_dtype():
    from traceml_b200.instrumentation.layers import LAYER_RECORD_DTYPE

    return LAYER_RECORD_DTYPE


def make_records(steps: List[int], n_layers: int, rng: np.random.Generator, *, fwd_calls=None, bwd_calls=None,
                 ns_choices=None) -> np.ndarray:
    """``[len(steps), n_layers]`` records; ``ns_choices`` (optional) draws durations from a small
    set, so equal times -- and worst-rank / sort ties -- happen."""
    recs = np.zeros((len(steps), n_layers), dtype=layer_dtype())
    recs["step"] = np.asarray(steps, dtype=np.uint64)[:, None]
    shape = recs.shape
    if ns_choices is None:
        recs["fwd_ns"] = rng.integers(1_000, 5_000_000, size=shape)
        recs["bwd_ns"] = rng.integers(1_000, 9_000_000, size=shape)
    else:
        recs["fwd_ns"] = rng.choice(np.asarray(ns_choices, dtype=np.uint64), size=shape)
        recs["bwd_ns"] = rng.choice(np.asarray(ns_choices, dtype=np.uint64), size=shape)
    recs["fwd_calls"] = 1 if fwd_calls is None else fwd_calls
    recs["bwd_calls"] = 1 if bwd_calls is None else bwd_calls
    recs["fwd_ns"][recs["fwd_calls"] == 0] = 0
    recs["bwd_ns"][recs["bwd_calls"] == 0] = 0
    return recs


# ------------------------------------------------------------------------------ restatement
def restate(records: Dict[int, np.ndarray], world: int) -> Dict[str, Any]:
    """Per-layer values of one tick from each rank's retained records (commit order)."""
    last = {}
    for r in range(world):
        rec = records.get(r)
        if rec is None or not len(rec):
            continue
        f = np.flatnonzero((rec["fwd_calls"] > 0).any(axis=1))
        b = np.flatnonzero((rec["bwd_calls"] > 0).any(axis=1))
        if len(f) and len(b):
            last[r] = min(int(rec["step"][f[-1], 0]), int(rec["step"][b[-1], 0]))
    if not last:
        return {"safe_step": None}
    safe = min(last.values())
    n_layers = next(len(v[0]) for v in records.values() if v is not None and len(v))
    cur = np.zeros((2, n_layers))
    peak = np.zeros((2, n_layers))
    has_cur = np.zeros((2, n_layers), bool)
    has_peak = np.zeros((2, n_layers), bool)
    rank_cur = {d: {} for d in (0, 1)}  # d -> rank -> [n_layers] current (nan: absent)
    missing = set()
    for d, (ns, calls) in enumerate((("fwd_ns", "fwd_calls"), ("bwd_ns", "bwd_calls"))):
        for r in range(world):
            rec = records.get(r)
            rows = [] if rec is None or not len(rec) else list(np.flatnonzero((rec[calls] > 0).any(axis=1)))
            lo = 0
            for k, i in enumerate(rows):
                if int(rec["step"][i, 0]) < safe:
                    lo = k + 1
            window = rows[lo:]
            at = [i for i in window if int(rec["step"][i, 0]) == safe]
            if not at:
                missing.add(r)
                continue
            c = at[-1]
            ms = lambda i: np.array([float(int(x)) / 1.0e6 for x in rec[ns][i]])  # noqa: E731
            present = rec[calls][c] > 0
            vals = ms(c)
            rank_cur[d][r] = np.where(present, vals, np.nan)
            cur[d] = np.where(present, np.maximum(cur[d], vals), cur[d])
            has_cur[d] |= present
            for i in window:
                p = rec[calls][i] > 0
                peak[d] = np.where(p, np.maximum(peak[d], ms(i)), peak[d])
                has_peak[d] |= p
    worst = []
    for l in range(n_layers):
        totals: Dict[int, float] = {}
        for d in (0, 1):
            for r, v in rank_cur[d].items():
                if not np.isnan(v[l]):
                    totals[r] = totals.get(r, 0.0) + float(v[l])
        worst.append(max(totals.items(), key=lambda x: x[1])[0] if totals else None)
    return {"safe_step": safe, "missing_ranks": sorted(missing), "cur": cur, "peak": peak,
            "has_cur": has_cur, "has_peak": has_peak, "worst": worst}


def check_first_tick(got: Dict[str, Any], want: Dict[str, Any], names: List[str], world: int) -> None:
    """A first tick's result against the restatement (avg == current on a first tick)."""
    if want["safe_step"] is None:
        assert got["safe_step"] is None and got["all_items"] == [] and got["missing_ranks"] == list(range(world))
        assert got["status_message"] == "Waiting for timing data from all ranks."
        return
    assert got["safe_step"] == want["safe_step"]
    assert got["missing_ranks"] == want["missing_ranks"]
    assert got["incomplete"] == bool(want["missing_ranks"]) and got["world_size"] == world
    by = {r["layer"]: r for r in got["all_items"]}
    inside = want["has_peak"][0] | want["has_peak"][1]
    assert set(by) == {names[i] for i in np.flatnonzero(inside)}
    for i in np.flatnonzero(inside):
        row = by[names[i]]
        for d, tag in enumerate(("forward", "backward")):
            assert row[f"{tag}_current"] == want["cur"][d][i], (names[i], tag)
            assert row[f"{tag}_avg"] == want["cur"][d][i]
            assert row[f"{tag}_peak"] == want["peak"][d][i], (names[i], tag)
        assert row["worst_rank"] == want["worst"][i], names[i]
        assert row["total_current"] == row["forward_current"] + row["backward_current"]
    totals = [r["total_avg"] for r in got["all_items"]]
    assert totals == sorted(totals, reverse=True)


def check_top_n(got: Dict[str, Any], top_n: int) -> None:
    items = got["all_items"]
    assert got["top_items"] == items[:top_n]
    rest = items[top_n:]
    o = got["other"]
    assert o["total_forward_current"] == sum(r["forward_current"] for r in rest)
    assert o["total_backward_avg"] == sum(r["backward_avg"] for r in rest)
    assert o["pct"] == sum(r["pct"] for r in rest)


# ------------------------------------------------------------------------------ the reference
def reference_importable() -> bool:
    if os.path.isdir(REF_SRC) and REF_SRC not in sys.path:
        sys.path.append(REF_SRC)
        os.environ.setdefault("TRACEML_LOGS_DIR", os.path.join("/tmp", "traceml_ref_logs"))
    try:
        import traceml.renderers.layer_combined_time.compute  # noqa: F401

        return True
    except Exception:  # noqa: BLE001
        return False


def wire_rows(records: np.ndarray, names: List[str], device: int = 0) -> Dict[str, List[Dict[str, Any]]]:
    """``LayerProfile.wire_rows`` of the product, on records that did not come from hooks."""
    from traceml_b200.instrumentation.layers import LayerProfile

    stub = types.SimpleNamespace(names=list(names), seq=0, model_id=1,
                                 engine=types.SimpleNamespace(device=device))
    return LayerProfile.wire_rows(stub, records)


def reference_store(records: Dict[int, np.ndarray], names: List[str]):
    """The reference's in-memory remote store holding each rank's layer-time tables."""
    from traceml.database.remote_database_store import RemoteDBStore

    store = RemoteDBStore(max_rows=max([len(v) for v in records.values()] + [1]) + 1)
    for r, rec in records.items():
        if rec is None or not len(rec):
            continue
        rows = wire_rows(rec, names, device=r)
        for tag in ("forward", "backward"):
            store.ingest({"rank": r, "sampler": f"Layer{tag.capitalize()}TimeSampler",
                          "tables": {f"layer_{tag}_time": rows[f"layer_{tag}_time"]}})
    return store


def reference_computer(monkeypatch, world: int, **kw):
    from traceml.renderers.layer_combined_time import compute as ref

    monkeypatch.setattr(ref, "get_ddp_info", lambda: (world > 1, 0, world))
    return ref.LayerCombinedTimerData(remote_store=None, **kw)


def reference_tick(comp, records: Dict[int, np.ndarray], names: List[str]) -> Dict[str, Any]:
    import dataclasses

    comp._remote_store = reference_store(records, names)
    return dataclasses.asdict(comp.compute_display_data())


def assert_same_result(got: Dict[str, Any], want: Dict[str, Any], what: str = "") -> None:
    """Every field ``==``.  Rows whose ``total_avg`` ties come out of a Python set in the reference:
    their relative order is compared as a set."""
    for k in ("safe_step", "incomplete", "missing_ranks", "world_size", "status_message", "other"):
        assert got[k] == want[k], (what, k, got[k], want[k])
    for k in ("all_items", "top_items"):
        a, b = got[k], want[k]
        assert len(a) == len(b), (what, k)
        assert [r["total_avg"] for r in a] == [r["total_avg"] for r in b], (what, k)
        key = lambda r: (-r["total_avg"], r["layer"])  # noqa: E731
        assert sorted(a, key=key) == sorted(b, key=key), (what, k)


# ------------------------------------------------------------------------------ seeded rings
SEEDED = ("staggered", "duplicates", "fwd_only_layer", "eval_step", "no_bwd_rank", "no_bwd_single",
          "missing_safe", "ties", "wrapped")


def seeded(name: str, n_layers: int, seed: int = 0):
    """-> (world, {rank: records in commit order}, ring_steps).  The records a ring of
    ``ring_steps`` retains are ``records[-ring_steps:]``."""
    rng = np.random.default_rng(seed + 1000 * SEEDED.index(name) + n_layers)
    mk = lambda steps, **kw: make_records(steps, n_layers, rng, **kw)  # noqa: E731
    ring = 64
    if name == "staggered":      # different newest steps: safe = 37, the peaks see newer steps
        recs = {0: mk(list(range(1, 41))), 1: mk(list(range(1, 38))), 2: mk(list(range(5, 46)))}
    elif name == "duplicates":   # re-run steps keep their id: the newest row of an id wins
        recs = {0: mk([1, 2, 3, 3, 4, 4, 5, 5, 5]), 1: mk([1, 2, 2, 3, 4, 5, 6])}
    elif name == "fwd_only_layer":
        bc = np.ones((20, n_layers), np.uint32)
        bc[:, 0] = 0
        recs = {0: mk(list(range(1, 21)), bwd_calls=bc), 1: mk(list(range(1, 21)), bwd_calls=bc)}
    elif name == "eval_step":    # rank 1's newest step is forward only: it pulls the safe step back
        bc = np.ones((12, n_layers), np.uint32)
        bc[-1] = 0
        recs = {0: mk(list(range(1, 13))), 1: mk(list(range(1, 13)), bwd_calls=bc)}
    elif name == "no_bwd_rank":  # rank 1 never has a backward row: missing, ranks 0 and 2 set the step
        recs = {0: mk(list(range(1, 11))), 1: mk(list(range(1, 9)), bwd_calls=0), 2: mk(list(range(1, 12)))}
    elif name == "no_bwd_single":
        recs = {0: mk(list(range(1, 6)), bwd_calls=0)}
    elif name == "missing_safe":  # rank 2 skipped step 9 (= the safe step): incomplete
        recs = {0: mk(list(range(1, 10))), 1: mk(list(range(1, 12))),
                2: mk([s for s in range(1, 12) if s != 9])}
    elif name == "ties":         # identical rings: every worst rank ties, totals tie across layers
        one = mk(list(range(1, 9)), ns_choices=[1000, 2000, 3000])
        recs = {r: one.copy() for r in range(4)}
    elif name == "wrapped":      # the ring turned over several times; only its last 16 steps count
        ring = 16
        recs = {0: mk(list(range(1, 71))), 1: mk(list(range(1, 66)))}
    else:
        raise KeyError(name)
    return len(recs), recs, ring


def retained(recs: Dict[int, np.ndarray], ring: int) -> Dict[int, np.ndarray]:
    return {r: v[-ring:] for r, v in recs.items()}
