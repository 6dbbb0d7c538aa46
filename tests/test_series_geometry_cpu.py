"""CPU companion of test_gpu_series_geometry.py: the numpy restatements it compares the kernels with,
and proof that its data can tell a right kernel from a plausibly wrong one.

* the ring geometries put the seam, the tail and t_start where the window pass is most likely to
  break (asserted, so an edit of the table cannot quietly lose a case);
* the restatement of the window pass's counters agrees with the row-level oracles, on rings that
  repeat step ids behind unusable rows at the seam, across tile edges and across t_start;
* teeth: on the GPU tests' own inputs, a sequential rank sum differs from numpy's blocked pairwise
  sum (K7d), the two middle values of an even rank count differ (K4, K7d), and a window pass whose
  halo is off by one slot at the seam, or that misses a duplicate at a tile edge, reports other
  candidate counts or another density verdict.
"""
import numpy as np
import pytest

import series_geometry as sg
from helpers import oracle_time_rows

# the H100 SXM's 132 SMs x 2 CTAs x 8 warps x 32 rows: the rows one trip of the window pass covers
TRIP_ROWS = 132 * 2 * 8 * 32


def _lane(slots, commits):
    i0 = sg.seam_row(slots, commits)
    return None if i0 is None else i0 % sg.TILE


def test_geometries_cover_the_tile_edges():
    lanes, tails, ns = set(), set(), set()
    for name, (slots, commits, W) in sg.GEOMETRIES.items():
        n = sg.retained(slots, commits)
        ns.add(n)
        tails.add(n % 32)
        if commits > slots:
            assert commits > 5 * slots, name
            lanes.add(_lane(slots, commits))
    assert {0, 1, 15, 30, 31} <= lanes
    assert {1, 17, 31} <= tails and {1, 31, 32, 33} <= ns
    assert any((sg.retained(s, c) - w) % 32 for s, c, w in sg.GEOMETRIES.values() if sg.retained(s, c) > w)
    assert sum(1 for s, c, _ in sg.GEOMETRIES.values() if s % 2 == 1 and c > 5 * s) >= 6
    slots, commits, W = sg.GEOMETRIES["big_seam17"]
    assert W > 2 * TRIP_ROWS and _lane(slots, commits) == 17
    # the seam falls where it is documented
    assert sg.seam_row(65, 6 * 65 + 33) == 32 and sg.seam_row(4113, 6 * 4113 + 2066) == 2047
    rs = sg.row_slots(4113, 6 * 4113 + 2066)
    assert rs[2046] == 4112 and rs[2047] == 0
    for name, (slots, commits, W) in sg.CHAIN_GEOMETRIES.items():
        n = sg.retained(slots, commits)
        assert W > (1 << 17) and n > W and (n - W) % 32 != 0, name
        assert _lane(slots, commits) not in (None, 0), name


@pytest.mark.parametrize("name", list(sg.ADVERSARIAL_RINGS))
def test_adversarial_pairs_sit_where_named(name):
    slots, commits, W = sg.GEOMETRIES[name]
    n = sg.retained(slots, commits)
    t0 = n - W
    pairs = sg.adversarial_pairs(name)
    assert pairs["tile_edge"] % 32 == 31 and pairs["tile_edge"] >= t0
    rs = sg.row_slots(slots, commits)
    assert rs[pairs["seam"]] == slots - 1 and rs[pairs["seam"] + 1] == 0
    assert pairs["t_start"] + 1 == t0 and pairs["window_head"] == t0 and pairs["window_tail"] + 2 == n
    base = sg.step_records(n, 5)
    for label, a in pairs.items():
        for no_mem in (False, True):
            recs = sg.with_duplicate_and_hole(base, a, sg.hole_for(name, a), no_mem)
            c = sg.window_counters(recs, W)
            steps = recs["step"].astype(np.int64)
            # the trap: as many ids spanned as there are rows, yet one id twice
            assert steps[-1] - steps[0] + 1 == n and len(np.unique(steps)) == n - 1, label
            assert c["dup_rows"] == 1 and c["monotone"] and c["ok"] == 0, (label, c)
            assert c["n_cand"][1] == n - 1, (label, c)


def test_decreases_are_counted():
    base = sg.step_records(4113, 3)
    for rows in ([2047], [3200], [2047, 3200]):
        c = sg.window_counters(sg.with_decreases(base, rows), 3001)
        assert c["violations"] == len(rows) and c["monotone"] == 0 and c["dup_rows"] == 0


# ----------------------------------------------------------------------------- restatement vs row oracles
@pytest.mark.parametrize("name,mode,seed", [("n1025_seam15", "mixed", 11), ("n4113_seam31", "mixed", 12),
                                            ("n8191_seam0", "mixed", 13), ("n8191_seam0", "dense", 14),
                                            ("n4113_seam31", "mixed", 104), ("n8191_seam0", "mixed", 105)])
def test_restated_time_candidates_match_row_level_oracle(name, mode, seed):
    """One rank: the time candidates are the window's aligned steps (common suffix of one rank)."""
    from oracle import step_memory_oracle, step_time_oracle
    from helpers import oracle_mem_rows

    recs, slots, commits, W = sg.ring_records(name, seed, mode)
    c = sg.window_counters(recs, W)
    o = step_time_oracle.step_time_section(oracle_time_rows({0: recs}, W), max_rows=W)
    win = o["data"]["aligned_window"]
    assert win["steps_analyzed"] == c["n_cand"][0]
    assert (win["start_step"], win["end_step"]) == (c["lo"][0], c["hi"][0])
    assert o["data"]["latest_step_observed"] == c["latest_step"]
    # memory over every retained row: one candidate per step id that has a row with memory
    m = step_memory_oracle.step_memory_section(oracle_mem_rows({0: recs}), window_size=len(recs))
    steps = m["window"]["steps"]
    assert len(steps) == c["n_cand"][1]
    assert (min(steps), max(steps)) == (c["lo"][1], c["hi"][1])
    if mode == "mixed":
        assert c["dup_rows"] > 0 and c["n_cand"][0] < c["n_win"] and not c["ok"]
        # the planted repeats behind unusable rows: taking the oldest row of a step, usable or not,
        # loses steps the reference keeps
        assert sg.planted_runs(slots, commits, W)
        assert sg.window_counters(recs, W, rule="fused")["n_cand"][0] < c["n_cand"][0]
    else:
        assert c["ok"] and c["n_both"] == c["n_win"]
        assert sg.window_counters(recs, W, rule="fused") == c


# ----------------------------------------------------------------------------- teeth: window pass
def _halo_prev(recs, slots, commits, rows, offset):
    """prev step ids as a pass sees them whose lane-0 halo, at ``rows``, reads the ring ``offset`` slots
    off the right one (the slot before the tile)."""
    prev, _, _ = sg.neighbours(recs)
    prev = prev.copy()
    rs = sg.row_slots(slots, commits)
    by_slot = np.empty(slots, dtype=np.uint64)
    by_slot[rs] = recs["step"]
    for i in rows:
        prev[i] = by_slot[(rs[i] - 1 + offset) % slots]
    return prev


@pytest.mark.parametrize("name", ["seam0", "n8191_seam0"])
def test_teeth_halo_shifted_at_the_seam(name):
    recs, slots, commits, W = sg.ring_records(name, 21)
    i0 = sg.seam_row(slots, commits)
    assert i0 % 32 == 0 and i0 > max(0, len(recs) - W)
    good = sg.window_counters(recs, W)
    assert good["ok"]
    # the halo read from the tile's own first slot: the seam row looks like a repeat of itself
    bad = sg.window_counters(recs, W, prev_step=_halo_prev(recs, slots, commits, [i0], +1))
    assert bad["n_cand"][0] == good["n_cand"][0] - 1 and bad["dense"][0] == 0 and bad["dup_rows"] == 1
    # a duplicate across the seam: the halo one slot too far back misses it and accepts the window
    dup = sg.with_duplicate_and_hole(recs, i0 - 1, sg.hole_for(name, i0 - 1))
    good = sg.window_counters(dup, W)
    bad = sg.window_counters(dup, W, prev_step=_halo_prev(dup, slots, commits, [i0], -1))
    assert good["dense"][0] == 0 and bad["dense"][0] == 1
    assert bad["n_cand"][0] == good["n_cand"][0] + 1


@pytest.mark.parametrize("name", list(sg.ADVERSARIAL_RINGS))
@pytest.mark.parametrize("no_mem", [False, True])
def test_teeth_duplicate_missed_at_a_tile_edge(name, no_mem):
    slots, commits, W = sg.GEOMETRIES[name]
    n = sg.retained(slots, commits)
    a = sg.adversarial_pairs(name)["tile_edge"]
    recs = sg.with_duplicate_and_hole(sg.step_records(n, 5), a, sg.hole_for(name, a), no_mem)
    good = sg.window_counters(recs, W)
    prev, nxt, nfl = sg.neighbours(recs)
    prev, nxt = prev.copy(), nxt.copy()
    prev[a + 1] = recs["step"][a + 1] - 1        # lane 0 of the next tile: halo not read
    nxt[a] = recs["step"][a] + 1                 # lane 31: halo not read
    bad = sg.window_counters(recs, W, prev_step=prev, next_step=nxt, next_flags=nfl)
    assert good["ok"] == 0 and good["dense"] == [0, 0]
    assert bad["n_cand"][0] == good["n_cand"][0] + 1 and bad["dense"][0] == 1
    if not no_mem:   # the older row of the pair becomes a memory candidate too: the window is accepted
        assert bad["n_cand"][1] == good["n_cand"][1] + 1 and bad["ok"] == 1


# ----------------------------------------------------------------------------- teeth: K4 / K7d
def _pairwise(v):
    """numpy's pairwise_sum restated for fewer than 128 contiguous f64: a plain loop below 8, else
    eight running partials combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remainder."""
    n = len(v)
    if n < 8:
        s = 0.0
        for x in v:
            s += x
        return s
    r = [float(x) for x in v[:8]]
    i = 8
    while i + 8 <= n:
        for k in range(8):
            r[k] += float(v[i + k])
        i += 8
    s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for x in v[i:]:
        s += float(x)
    return s


def _sequential(v):
    s = 0.0
    for x in v:
        s += float(x)
    return s


@pytest.mark.parametrize("R", range(1, 65))
def test_numpy_sum_order_and_comb_expected(R):
    """np.sum of a 1-D rank array is the blocked pairwise order above, and comb_expected's
    vectorised sum is np.sum of each step's own 1-D array."""
    rows = sg.rank_rows(R, 1000, seed=700 + R)
    for first, k in sg.COMB_COLS:
        exp = sg.comb_expected(rows, first, k)
        for m in range(k):
            for j in range(0, 1000, 37):
                v = np.ascontiguousarray(rows[:, j, first + m])
                assert exp[m, 2, j] == np.sum(v) == _pairwise(v), (R, first, m, j)
                assert exp[m, 0, j] == np.median(v) and exp[m, 1, j] == np.max(v)


@pytest.mark.parametrize("R", range(8, 65))
def test_teeth_sequential_sum_differs(R):
    rows = sg.rank_rows(R, 1000, seed=700 + R)
    diff = total = 0
    for first, k in sg.COMB_COLS:
        exp = sg.comb_expected(rows, first, k)
        for m in range(k):
            for j in range(1000):
                diff += _sequential(rows[:, j, first + m]) != exp[m, 2, j]
                total += 1
    assert diff >= 0.1 * total, (R, diff, total)


@pytest.mark.parametrize("R", range(2, 65, 2))
def test_teeth_even_rank_middles_differ(R):
    """Taking v[R/2] (or v[R/2 - 1]) for an even R would change most medians: K4's 16 series
    (the K4 seed) and K7d's raw columns (the K7d seed)."""
    from oracle import fast_oracle

    for seed in (500 + R, 700 + R):
        rows = sg.rank_rows(R, 1000, seed=seed)
        f, b, o = rows[:, :, 2], rows[:, :, 3], rows[:, :, 4]
        compute = (f + b) + o
        traced = np.maximum(rows[:, :, 5], compute)
        cols = [rows[:, :, 0], f, b, o, traced, np.maximum(0.0, traced - compute), rows[:, :, 6], rows[:, :, 7]]
        v = np.sort(np.stack(cols), axis=1)            # [metric, R, n]
        lo, hi = v[:, R // 2 - 1, :], v[:, R // 2, :]
        assert np.mean(lo != hi) > 0.5, (R, seed, float(np.mean(lo != hi)))
        med = fast_oracle.series16(rows)[0::2]
        assert np.mean(med != hi) > 0.5 and np.mean(med != lo) > 0.5
