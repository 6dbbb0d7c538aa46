"""GPU: the window pass and the per-step series kernels at every ring seam, tile edge and rank count.

Everything compared here is exact -- ns -> ms is correctly rounded; median, max, numpy's pairwise
sum, the integer counters and the u64 byte sums are exact operations -- so the kernels must equal
their numpy restatements (tests/series_geometry.py) byte for byte:

* the single-rank window pass, fused (``k_window_fused``, called directly at any size) and staged
  (``k_window_rows`` + the dense selection), on rings whose seam falls on lanes 0, 1, 15, 17, 30 and
  31 of a warp tile, with tails of 1, 17 and 31 rows, unaligned window starts and a window long
  enough that every warp makes three or more trips; every counter of ``tml_win_info``, the series,
  the exact byte sums and maxima, and the tree sums (rel 1e-13 of math.fsum, DESIGN.md section 3);
* dense-looking windows that hide one duplicated step id behind one hole, with the pair on a tile
  edge, across the seam, across t_start and at either end of the window: never accepted, and the
  full build agrees with the row-level oracles; a step id logged again after a row with nothing to
  summarise: the staged pass keeps the step through its oldest usable row, as the reference does;
  step ids that decrease across the seam or a tile edge: the same error from both passes, with the
  exact count;
* the chained single-rank build on windows just above its 2^17-row threshold;
* K4 (``k_window_reduce<R>`` / ``k_window_reduce_any``) and K7d (``k_comb_series``) for every rank
  count 1..64, including K4's sharded writes, its time-only / memory-only masks and its argument checks.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import series_geometry as sg
from helpers import build_vs_row_oracles

pytestmark = pytest.mark.gpu

SENTINEL = np.uint64(0x7FF4_DEAD_BEEF_0001)   # a NaN payload no kernel computes
GUARD = 4096                                  # values past the end of every output that must stay untouched
TML_ERR_ARG = -2
SEEDS = {name: 100 + i for i, name in enumerate({**sg.GEOMETRIES, **sg.CHAIN_GEOMETRIES})}


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def reducer(cuda):
    """A context for the K4 / K7d calls (their inputs are device pointers of our own)."""
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=64, proc_slots=64)
    yield eng
    eng.close()


def _buffer(n_values):
    return torch.from_numpy(np.full(n_values + GUARD, SENTINEL, dtype=np.uint64).view(np.float64)).cuda()


def _host(buf, n_values):
    """(the first n_values as f64, whether the guard tail still holds the sentinel)"""
    h = buf.cpu().numpy()
    return h[:n_values].copy(), bool((h[n_values:].view(np.uint64) == SENTINEL).all())


def _is_sentinel(a):
    return bool((np.ascontiguousarray(a).view(np.uint64) == SENTINEL).all())


def _ring(recs, slots, commits):
    """An engine whose ring has taken ``commits`` records and retains ``recs`` (its last ones)."""
    from traceml_b200.engine import Engine
    from traceml_b200.records import STEP_RECORD_DTYPE

    eng = Engine(device=0, rank=0, world=1, ring_slots=slots, proc_slots=64)
    left = commits - len(recs)
    filler = np.zeros(min(max(left, 0), slots), dtype=STEP_RECORD_DTYPE)
    while left > 0:   # overwritten by what follows: it only advances the ring
        k = min(left, len(filler))
        eng.load_steps(filler[:k])
        torch.cuda.synchronize()
        left -= k
    eng.load_steps(recs)
    torch.cuda.synchronize()
    assert eng.step_count == commits
    return eng


def _fused(eng, window, n_win):
    """tml_win_fused into a sentinel-filled buffer: (status, WinInfo, AlignInfo, ok, series [16, n_win], guard ok)"""
    from traceml_b200 import _abi

    buf = _buffer(16 * n_win)
    info, al, ok = _abi.WinInfo(), _abi.AlignInfo(), C.c_uint32(7)
    rc = _abi.lib().tml_win_fused(eng.handle, int(window), buf.data_ptr(), 0, C.byref(info), C.byref(al), C.byref(ok))
    torch.cuda.synchronize()
    ser, guard = _host(buf, 16 * n_win)
    return rc, info, al, int(ok.value), ser.reshape(16, n_win), guard


def _counters(info):
    return {"n_retained": int(info.n_retained), "latest_step": int(info.latest_step), "monotone": int(info.monotone),
            "dup_rows": int(info.dup_rows), "n_rows": list(info.n_rows), "n_cand": list(info.n_cand),
            "lo": list(info.lo), "hi": list(info.hi), "t_count": int(info.t_count), "n_both": int(info.n_both),
            "dense": list(info.dense)}


def _restated(c):
    return {k: c[k] for k in ("n_retained", "latest_step", "monotone", "dup_rows", "n_rows", "n_cand", "lo", "hi",
                              "t_count", "n_both", "dense")}


def _expected_series(recs, window):
    from oracle import fast_oracle

    return fast_oracle.series16(fast_oracle.window_rows(recs[max(0, len(recs) - window):])[None])


def _check_sums(info, al, ok, recs, window):
    """Tree sums against math.fsum; with ok, the aligned sums: exact integer byte sums and maxima."""
    for k, addends in enumerate(sg.tree_sum_addends(recs, window)):
        ref = math.fsum(addends.tolist())
        assert abs(info.t_sums[k] - ref) <= 1e-13 * abs(ref), (k, info.t_sums[k], ref)
    if ok:
        w = recs[max(0, len(recs) - window):]
        pa = [int(x) for x in w["peak_alloc"]]
        pr = [int(x) for x in w["peak_resv"]]
        assert list(al.m_sums) == [float(sum(pa)), float(sum(pr)), float(max(pa)), float(max(pr))]
        t = list(info.t_sums)
        t[4] = t[5]   # aligned step_cpu = sum of traced (alignment.py:72)
        assert list(al.t_sums) == t


# ----------------------------------------------------------------------------- 1. window pass geometry
@pytest.mark.parametrize("mode", ["dense", "mixed"])
@pytest.mark.parametrize("name", list(sg.GEOMETRIES))
def test_window_pass_geometry(cuda, name, mode):
    from oracle import fast_oracle
    from traceml_b200 import _abi

    recs, slots, commits, W = sg.ring_records(name, SEEDS[name], mode)
    c = sg.window_counters(recs, W)
    cf = sg.window_counters(recs, W, rule="fused")
    assert cf["ok"] == c["ok"]
    if mode == "dense":
        assert c["ok"] == 1
    eng = _ring(recs, slots, commits)
    try:
        rc, info, al, ok, ser, guard = _fused(eng, W, c["n_win"])
        assert rc == 0, _abi.lib().tml_last_error()
        assert _counters(info) == _restated(cf)
        assert ok == c["ok"]
        assert guard, "the fused pass wrote past its 16 x n_window series"
        assert ser.tobytes() == _expected_series(recs, W).tobytes()
        _check_sums(info, al, ok, recs, W)
        if ok:
            assert (al.n_common, al.start_step, al.end_step, al.n_rows) == (c["n_win"], c["lo"][0], c["hi"][0], c["n_win"])

        # the staged pass over the same ring: same counters, and the dense window's aligned rows
        info2 = eng.win_prepare(W)
        assert _counters(info2) == _restated(c)
        if info2.dense[0]:
            al2 = eng.win_select_dense(_abi.KIND_TIME, c["lo"][0], c["n_cand"][0])
            rows = eng.win_rows_tensor(_abi.KIND_TIME, c["n_win"]).cpu().numpy().reshape(c["n_win"], 8)
            torch.cuda.synchronize()
            assert rows.tobytes() == fast_oracle.window_rows(recs[c["t_start"]:]).tobytes()
            w = recs[c["t_start"]:]
            assert list(al2.m_sums[:2]) == [float(sum(int(x) for x in w["peak_alloc"])),
                                            float(sum(int(x) for x in w["peak_resv"]))]
            assert list(al2.m_sums[2:]) == [float(int(w["peak_alloc"].max())), float(int(w["peak_resv"].max()))]
    finally:
        eng.close()


# ----------------------------------------------------------------------------- adversarial acceptance
@pytest.mark.parametrize("no_mem", [False, True], ids=["both_mem", "newer_without_mem"])
@pytest.mark.parametrize("where", ["tile_edge", "seam", "t_start", "window_head", "window_tail"])
@pytest.mark.parametrize("name", list(sg.ADVERSARIAL_RINGS))
def test_duplicate_behind_a_hole_is_never_dense(cuda, name, where, no_mem):
    from traceml_b200 import _abi

    slots, commits, W = sg.GEOMETRIES[name]
    n = sg.retained(slots, commits)
    a = sg.adversarial_pairs(name)[where]
    recs = sg.with_duplicate_and_hole(sg.step_records(n, 5), a, sg.hole_for(name, a), no_mem)
    c = sg.window_counters(recs, W)
    assert c["dup_rows"] == 1 and c["ok"] == 0
    assert sg.window_counters(recs, W, rule="fused") == c   # every row usable: the two rules agree
    eng = _ring(recs, slots, commits)
    try:
        rc, info, al, ok, ser, guard = _fused(eng, W, c["n_win"])
        assert rc == 0, _abi.lib().tml_last_error()
        assert ok == 0 and info.dup_rows == 1
        assert list(info.n_cand) == c["n_cand"] and list(info.dense) == c["dense"]
        assert _counters(info) == _restated(c)
        assert guard and ser.tobytes() == _expected_series(recs, W).tobytes()
        assert _counters(eng.win_prepare(W)) == _restated(c)
        build_vs_row_oracles(eng, recs, W)
    finally:
        eng.close()


@pytest.mark.parametrize("where", ["seam", "tile_edge", "both"])
@pytest.mark.parametrize("name", list(sg.ADVERSARIAL_RINGS))
def test_decreasing_step_ids(cuda, name, where):
    from traceml_b200 import _abi

    slots, commits, W = sg.GEOMETRIES[name]
    n = sg.retained(slots, commits)
    seam = sg.seam_row(slots, commits)
    edge = (sg.adversarial_pairs(name)["tile_edge"] + 1)   # lane 0: its previous row comes from the halo
    rows = {"seam": [seam], "tile_edge": [edge], "both": [seam, edge]}[where]
    recs = sg.with_decreases(sg.step_records(n, 3), rows)
    c = sg.window_counters(recs, W)
    assert c["violations"] == len(rows)
    eng = _ring(recs, slots, commits)
    try:
        rc, info, _, ok, _, guard = _fused(eng, W, c["n_win"])
        assert rc == _abi.TML_ERR_NONMONOTONIC and ok == 0 and guard
        msg = _abi.lib().tml_last_error().decode()
        assert f"({len(rows)} places)" in msg, msg
        assert info.monotone == 0
        with pytest.raises(_abi.TraceMLNativeError, match=rf"\({len(rows)} places\)"):
            eng.win_prepare(W)
    finally:
        eng.close()


# a step id logged again after a row with nothing to summarise (only h2d > 0): the time candidate is
# the step's oldest usable row in the window (the reference's choice), wherever the rows fall
REPEAT_CASES = {
    ("seam0", "in_tile"): [(20, (False, True))],
    ("seam0", "tile_edge_and_seam"): [(31, (False, True))],          # rows 31 | 32: lane 31 | lane 0, slot 64 | 0
    ("seam0", "two_unusable_across_edge"): [(30, (False, False, True))],
    ("seam0", "usable_unusable_usable"): [(30, (True, False, True))],
    ("seam0", "across_t_start"): [(14, (True, False, True))],       # t_start = 15
    ("n8191_seam0", "long_run_across_tiles"): [(4090, (False,) * 40 + (True,))],
    ("n8191_seam0", "planted"): sg.planted_runs(*sg.GEOMETRIES["n8191_seam0"]),
}


@pytest.mark.parametrize("name,label", list(REPEAT_CASES))
def test_repeated_step_after_unusable_row(cuda, name, label):
    from traceml_b200 import _abi

    slots, commits, W = sg.GEOMETRIES[name]
    recs = sg.with_repeats(sg.step_records(sg.retained(slots, commits), 9), REPEAT_CASES[(name, label)])
    c = sg.window_counters(recs, W)
    w = recs[c["t_start"]:]
    usable = (w["dur_ns"][:, sg.USABLE_COLS] > 0).any(axis=1)
    assert c["n_cand"][0] == len(np.unique(w["step"][usable]))   # one candidate per step with a usable row
    eng = _ring(recs, slots, commits)
    try:
        rc, info, _, ok, ser, guard = _fused(eng, W, c["n_win"])
        assert rc == 0 and ok == 0 and guard, _abi.lib().tml_last_error()
        assert _counters(info) == _restated(sg.window_counters(recs, W, rule="fused"))
        assert ser.tobytes() == _expected_series(recs, W).tobytes()
        assert _counters(eng.win_prepare(W)) == _restated(c)
        got = build_vs_row_oracles(eng, recs, W)
        assert got["step_time"]["data"]["aligned_window"]["steps_analyzed"] == c["n_cand"][0]
    finally:
        eng.close()


# ----------------------------------------------------------------------------- chained build
@pytest.mark.parametrize("name", list(sg.CHAIN_GEOMETRIES))
def test_chained_build_seam_inside_a_tile(cuda, name):
    import replay
    from traceml_b200 import sections

    recs, slots, commits, W = sg.ring_records(name, SEEDS[name])
    c = sg.window_counters(recs, W)
    assert c["ok"] == 1 and c["n_win"] > (1 << 17)
    exp = _expected_series(recs, W)
    eng = _ring(recs, slots, commits)
    try:
        res = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, W)
        red = res["reduce"]
        assert red.fused_rows
        t = red.time.series.cpu().numpy().copy()
        m = red.mem.series.cpu().numpy().copy()
        assert t[:12].tobytes() == exp[:12].tobytes() and m[12:16].tobytes() == exp[12:16].tobytes()
        rc, info, al, ok, ser, guard = _fused(eng, W, c["n_win"])
        assert rc == 0 and ok == 1 and guard
        assert ser.tobytes() == exp.tobytes()
        assert _counters(info) == _restated(c)
        _check_sums(info, al, ok, recs, W)
        assert res["step_time"]["data"]["aligned_window"]["steps_analyzed"] == c["n_win"]
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 2. K4 at every rank count
@pytest.mark.parametrize("R", range(1, 65))
def test_k4_every_rank_count(reducer, R):
    from oracle import fast_oracle
    from traceml_b200 import _abi

    both = _abi.MASK_TIME | _abi.MASK_MEM
    for n in sg.K4_SIZES:
        rows = sg.rank_rows(R, n, seed=500 + R if n == 1000 else 900 + R)
        dev = [torch.from_numpy(np.ascontiguousarray(rows[r])).cuda() for r in range(R)]
        exp = fast_oracle.series16(rows)

        buf = _buffer(16 * n)
        reducer.win_reduce(dev, both, n, 0, n, buf)
        torch.cuda.synchronize()
        full, guard = _host(buf, 16 * n)
        assert guard
        assert full.tobytes() == exp.tobytes(), (R, n)

        # R shards [g n / R, (g + 1) n / R) into one buffer, as the drivers split the steps
        buf = _buffer(16 * n)
        for g in range(R):
            reducer.win_reduce(dev, both, n, g * n // R, (g + 1) * n // R, buf)
        torch.cuda.synchronize()
        sharded, guard = _host(buf, 16 * n)
        assert guard and sharded.tobytes() == full.tobytes(), (R, n)

        for mask, on, off in ((_abi.MASK_TIME, slice(0, 12), slice(12, 16)),
                              (_abi.MASK_MEM, slice(12, 16), slice(0, 12))):
            buf = _buffer(16 * n)
            reducer.win_reduce(dev, mask, n, 0, n, buf)
            torch.cuda.synchronize()
            got, guard = _host(buf, 16 * n)
            got = got.reshape(16, n)
            assert guard and _is_sentinel(got[off]), (R, n, mask)
            assert got[on].tobytes() == exp[on].tobytes(), (R, n, mask)


def test_k4_rank_count_arguments(reducer):
    from traceml_b200 import _abi

    lib = _abi.lib()
    n = 100
    rows = [torch.zeros(n * 8, dtype=torch.float64, device="cuda") for _ in range(2)]
    buf = _buffer(16 * n)
    a = _abi.ReduceArgs()
    a.mask, a.n_common, a.shard_lo, a.shard_hi, a.series = 3, n, 0, n, buf.data_ptr()
    for i in range(_abi.TML_MAX_RANKS):
        a.rows[i] = rows[i % 2].data_ptr()
    for bad in (0, _abi.TML_MAX_RANKS + 1):   # the rows array holds 64 pointers: 65 must be refused
        a.n_ranks = bad
        assert lib.tml_win_reduce(reducer.handle, C.byref(a), 0) == TML_ERR_ARG, bad
    with pytest.raises(_abi.TraceMLNativeError, match=r"\(-2\)"):
        reducer.win_reduce([], 3, n, 0, n, buf)
    a.n_ranks = _abi.TML_MAX_RANKS   # and 64 itself runs
    assert lib.tml_win_reduce(reducer.handle, C.byref(a), 0) == 0
    torch.cuda.synchronize()
    got, guard = _host(buf, 16 * n)
    assert guard and not np.isnan(got).any() and (got == 0.0).all()


# ----------------------------------------------------------------------------- 3. K7d at every rank count
@pytest.mark.parametrize("R", range(1, 65))
def test_k7d_every_rank_count(reducer, R):
    for n in sg.K4_SIZES:
        rows = sg.rank_rows(R, n, seed=700 + R if n == 1000 else 1100 + R)
        dev = [torch.from_numpy(np.ascontiguousarray(rows[r])).cuda() for r in range(R)]
        for first, k in sg.COMB_COLS:
            exp = sg.comb_expected(rows, first, k)
            buf = _buffer(k * 3 * n)
            reducer.combined_series([t.data_ptr() for t in dev], n, first, k, buf)
            torch.cuda.synchronize()
            got, guard = _host(buf, k * 3 * n)
            assert guard
            assert got.tobytes() == exp.tobytes(), (R, n, first, k)
