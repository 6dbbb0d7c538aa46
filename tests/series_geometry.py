"""Shared by test_gpu_series_geometry.py and test_series_geometry_cpu.py (test infrastructure).

* ring geometry: where each retained row sits in a wrapped step ring, and where the seam falls;
* a numpy restatement of the single-rank window pass (``k_window_rows`` / ``k_window_fused``):
  the kernels' own candidate rules and every counter they report in ``tml_win_info``;
* the inputs of the window-pass, K4 (``k_window_reduce``) and K7d (``k_comb_series``) tests, so the
  CPU teeth checks run on exactly the data the GPU tests feed the kernels.

The window pass reads the retained ring in 32-row warp tiles over the retained rows (not the window
rows).  A row's neighbours come from warp shuffles inside a tile and from two 8-byte ring reads at
the tile edges: lane 0 reads the slot before the tile, lane 31 the slot after it.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from traceml_b200.records import FLAG_HAS_MEM, STEP_RECORD_DTYPE

TILE = 32
# summarised phases: usable = any of dataloader, forward, backward, optimizer, step wall > 0 (h2d is not)
USABLE_COLS = [0, 2, 3, 4, 5]


# ----------------------------------------------------------------------------- ring geometry
def retained(slots: int, commits: int) -> int:
    return min(int(slots), int(commits))


def row_slots(slots: int, commits: int) -> np.ndarray:
    """Ring slot of each retained row, oldest first."""
    n = retained(slots, commits)
    return (int(commits) - n + np.arange(n, dtype=np.int64)) % int(slots)


def seam_row(slots: int, commits: int) -> Optional[int]:
    """The retained row that sits in slot 0 after the slot ``slots - 1`` (None: no wrap inside)."""
    s = row_slots(slots, commits)
    hit = np.nonzero((s[1:] == 0))[0]
    return int(hit[0]) + 1 if hit.size else None


# name: (ring slots, commits, window).  Every ring but "unwrapped" has wrapped more than five times.
# The comments give the retained row count n, where the seam falls in its warp tile, and t_start.
GEOMETRIES: Dict[str, Tuple[int, int, int]] = {
    "n1": (1, 7, 1),                                   # n = 1
    "n31_seam30": (31, 6 * 31 + 1, 31),                # n = 31, seam on lane 30
    "n32_seam17": (32, 6 * 32 + 15, 20),               # n = 32, seam on lane 17, t_start = 12
    "n33_seam1": (33, 7 * 33 + 32, 33),                # n = 33 (n % 32 = 1), seam on lane 1
    "unwrapped": (65, 33, 40),                         # n = 33, ring not full, window wider than the ring
    "seam0": (65, 6 * 65 + 33, 50),                    # seam on lane 0 (tile starts at slot 0), t_start = 15
    "n1025_seam15": (1025, 6 * 1025 + 1010, 1000),     # n % 32 = 1, seam on lane 15, t_start = 25
    "n4113_seam31": (4113, 6 * 4113 + 2066, 3001),     # n % 32 = 17, seam on lane 31, t_start = 1112
    "n8191_seam0": (8191, 6 * 8191 + 4095, 5000),      # n % 32 = 31, seam on lane 0, t_start = 3191
    # > 2 x (2 CTAs/SM x 132 SMs x 8 warps x 32 rows) rows: every warp makes three or more trips
    "big_seam17": (300_001, 5 * 300_001 + 149_968, 299_990),   # seam on lane 17, t_start = 11
}

# windows just above 2^17 rows (the native build's bulk threshold), seam inside a tile, t_start % 32 != 0
CHAIN_GEOMETRIES: Dict[str, Tuple[int, int, int]] = {
    "chain_a": (131_201, 6 * 131_201 + 65_555, 131_100),
    "chain_b": (140_003, 6 * 140_003 + 1_009, 131_073),
    "chain_c": (163_847, 7 * 163_847 + 100_000, 150_001),
}


# ----------------------------------------------------------------------------- step records
def step_records(n: int, seed: int, *, mode: str = "dense", first_step: int = 1000) -> np.ndarray:
    """``n`` StepRecords with consecutive step ids ("dense") or with holes, unusable rows, rows
    without memory and duplicated step ids ("mixed").  Durations are integer ns over 12 decades; the
    step wall lies above or below forward + backward + optimizer; peaks are u64 byte counts whose
    window sums exceed 2^53."""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, dtype=STEP_RECORD_DTYPE)
    dur = np.floor(10.0 ** rng.uniform(0.0, 12.0, size=(n, 6))).astype(np.uint64)
    zero = rng.random(n) < 0.03                                # compute = 0: wait = wall
    dur[zero, 2:5] = 0
    comp = dur[:, 2] + dur[:, 3] + dur[:, 4]
    below = (comp.astype(np.float64) * rng.uniform(0.2, 1.0, n)).astype(np.uint64)
    above = comp + np.floor(10.0 ** rng.uniform(0.0, 9.0, n)).astype(np.uint64)
    dur[:, 5] = np.where(rng.random(n) < 0.5, below, above)
    r["dur_ns"] = dur
    r["n_calls"] = 1
    r["peak_alloc"] = rng.integers(1 << 30, 1 << 40, n, dtype=np.uint64)
    r["peak_resv"] = r["peak_alloc"] + rng.integers(0, 1 << 34, n, dtype=np.uint64)
    r["flags"] = FLAG_HAS_MEM
    inc = np.ones(n, dtype=np.int64)
    if mode == "mixed":
        inc += rng.random(n) < 0.01                            # holes
        inc[rng.random(n) < 0.005] = 0                         # duplicated step ids
        unusable = rng.random(n) < 0.02                        # only h2d > 0: not usable
        dur = r["dur_ns"]
        dur[unusable] = 0
        dur[unusable, 1] = 7
        r["dur_ns"] = dur
        r["flags"][rng.random(n) < 0.03] = 0                   # no memory peaks
    elif mode != "dense":
        raise ValueError(mode)
    inc[0] = 0
    r["step"] = first_step + np.cumsum(inc)
    r["seq"] = np.arange(n)
    return r


def with_repeats(recs: np.ndarray, runs) -> np.ndarray:
    """``runs``: (a, pattern) -> rows a .. a + len(pattern) - 1 all carry row a's step id (later ids
    move down to stay consecutive) and memory; where ``pattern`` is False the row is unusable (only
    h2d > 0): a step logged again after a row with nothing to summarise."""
    out = recs.copy()
    inc = np.diff(out["step"].astype(np.int64), prepend=int(out["step"][0]))
    dur = out["dur_ns"]
    for a, pattern in runs:
        k = len(pattern)
        inc[a + 1:a + k] = 0
        out["flags"][a:a + k] |= FLAG_HAS_MEM
        for j, usable in enumerate(pattern):
            if not usable:
                dur[a + j] = 0
                dur[a + j, 1] = 7
    out["dur_ns"] = dur
    out["step"] = (int(recs["step"][0]) + np.cumsum(inc)).astype(np.uint64)
    return out


def planted_runs(slots: int, commits: int, window: int):
    """Repeated step ids behind unusable rows where the window pass is most likely to get them wrong:
    across the seam, across a tile edge with two unusable rows before the usable one (the older rows
    lie in the previous tile), a usable row before an unusable one across a tile edge, and across
    t_start.  Empty for rings of fewer than 128 rows."""
    n = retained(slots, commits)
    if n < 128:
        return []
    t0 = max(0, n - window)
    edge = ((t0 + (n - t0) // 2) // TILE) * TILE + TILE - 1      # lane 31
    runs = [(edge - 1, (False, False, True)), (edge + 2 * TILE - 1, (True, False, True))]
    i0 = seam_row(slots, commits)
    if i0 is not None and i0 >= 1 and abs(i0 - edge) > 4 and abs(i0 - edge - 2 * TILE) > 4:
        runs.append((i0 - 1, (False, True)))
    if t0 >= 1:
        runs.append((t0 - 1, (True, False, True)))
    return runs


def ring_records(name: str, seed: int, mode: str = "dense") -> Tuple[np.ndarray, int, int, int]:
    """(retained records, slots, commits, window) of a geometry; "mixed" rings also carry the
    ``planted_runs``."""
    slots, commits, W = {**GEOMETRIES, **CHAIN_GEOMETRIES}[name]
    recs = step_records(retained(slots, commits), seed, mode=mode)
    if mode == "mixed":
        recs = with_repeats(recs, planted_runs(slots, commits, W))
    return recs, slots, commits, W


def with_duplicate_and_hole(recs: np.ndarray, a: int, hole: int, newer_without_mem: bool = False) -> np.ndarray:
    """Dense records -> row a + 1 repeats row a's step id and row ``hole`` skips one, so the step ids
    still span exactly as many ids as there are rows."""
    out = recs.copy()
    n = len(out)
    idx = np.arange(n)
    out["step"] = recs["step"][0] + idx - (idx >= a + 1) + (idx >= hole)
    assert out["step"][a] == out["step"][a + 1]
    if newer_without_mem:
        out["flags"][a + 1] = 0
    return out


def with_decreases(recs: np.ndarray, rows: List[int]) -> np.ndarray:
    """Consecutive step ids, except that each row in ``rows`` is two ids below its predecessor."""
    out = recs.copy()
    idx = np.arange(len(out), dtype=np.int64)
    back = np.zeros(len(out), dtype=np.int64)
    for r in rows:
        back += 3 * (idx >= r)
    out["step"] = (int(recs["step"][0]) + 3 * len(rows) + idx - back).astype(np.uint64)
    return out


# dense windows with one duplicated step id and one hole, on two rings: the seam on lane 31 of its
# tile, and the seam on lane 0 (its lane-0 halo read wraps to the ring's last slot)
ADVERSARIAL_RINGS = ("n4113_seam31", "n8191_seam0")


def adversarial_pairs(name: str) -> Dict[str, int]:
    """Where the duplicated pair (rows a, a + 1) goes: label -> a."""
    slots, commits, W = GEOMETRIES[name]
    n = retained(slots, commits)
    t0 = max(0, n - W)
    i0 = seam_row(slots, commits)
    edge = ((t0 + (n - t0) // 3) // TILE) * TILE + TILE - 1   # lane 31 of one tile, lane 0 of the next
    return {"tile_edge": edge, "seam": i0 - 1, "t_start": t0 - 1, "window_head": t0, "window_tail": n - 2}


def hole_for(name: str, a: int) -> int:
    slots, commits, W = GEOMETRIES[name]
    n = retained(slots, commits)
    t0 = max(0, n - W)
    return t0 + ((n - t0) * 3) // 4 if a < t0 + (n - t0) // 2 else t0 + (n - t0) // 4 + 5


# ----------------------------------------------------------------------------- window pass restated
def neighbours(recs: np.ndarray):
    """The true previous step id, next step id and next flags of every row (0 past the ends)."""
    step = recs["step"].astype(np.uint64)
    flags = recs["flags"].astype(np.uint32)
    z = np.zeros(1, dtype=np.uint64)
    return (np.concatenate([z, step[:-1]]), np.concatenate([step[1:], z]),
            np.concatenate([flags[1:], np.zeros(1, dtype=np.uint32)]))


def window_counters(recs: np.ndarray, window: int, prev_step=None, next_step=None, next_flags=None,
                    rule: str = "staged") -> Dict:
    """What the single-rank window pass reports for the retained rows ``recs`` (oldest first):
    ``tml_win_info`` restated with the kernels' own candidate rules --
      time:   usable, inside the last ``window`` rows, and the oldest usable row of its step id there
              (``k_window_rows``, the reference's choice); ``rule="fused"``: the oldest row of its step
              id there, if usable (``k_window_fused``: the two differ only where a step id repeats, and
              the fused pass accepts no such window);
      memory: carries memory, and the next row has another step id or carries no memory.
    A step id's rows form a run of consecutive rows, cut at t_start.  ``prev_step`` / ``next_step`` /
    ``next_flags``: the neighbours as a kernel sees them (default the true ones; the teeth checks pass
    broken halos)."""
    n = len(recs)
    t_start = max(0, n - int(window))
    n_win = n - t_start
    step = recs["step"].astype(np.uint64)
    has_mem = (recs["flags"] & FLAG_HAS_MEM) != 0
    usable = (recs["dur_ns"][:, USABLE_COLS] > 0).any(axis=1)
    tp, tn, tf = neighbours(recs)
    prev_step = tp if prev_step is None else prev_step
    next_step = tn if next_step is None else next_step
    next_flags = tf if next_flags is None else next_flags
    i = np.arange(n)
    in_time = i >= t_start
    head = (i == t_start) | (i == 0) | (prev_step != step)     # first row of a run
    uit = usable & in_time
    if rule == "fused":
        cand_t = uit & head
    elif rule == "staged":
        before = np.cumsum(uit) - uit                            # usable window rows above this one
        run = np.cumsum(head) - 1
        cand_t = uit & (before == before[np.nonzero(head)[0]][run])
    else:
        raise ValueError(rule)
    last_m = (i == n - 1) | (next_step != step) | ((next_flags & FLAG_HAS_MEM) == 0)
    cand = [cand_t, has_mem & last_m]
    out = {"n_retained": n, "t_start": t_start, "n_win": n_win,
           "latest_step": int(step.max()) if n else 0,
           "violations": int(np.sum((i > 0) & (step < prev_step))),
           "dup_rows": int(np.sum((i > 0) & (step == prev_step))),
           "n_rows": [n_win, int(has_mem.sum())],
           "t_count": int(np.sum(usable & in_time)),
           "n_both": int(np.sum(cand[0] & cand[1])),
           "n_cand": [], "lo": [], "hi": [], "dense": []}
    out["monotone"] = int(out["violations"] == 0)
    rows_in = [n_win, n]
    for k in range(2):
        c = int(cand[k].sum())
        lo = int(step[cand[k]].min()) if c else 0
        hi = int(step[cand[k]].max()) if c else 0
        out["n_cand"].append(c)
        out["lo"].append(lo)
        out["hi"].append(hi)
        out["dense"].append(int(c > 0 and c == rows_in[k] and hi - lo + 1 == c))
    # the fused pass hands its series over only if both kinds are dense over the same steps
    out["ok"] = int(out["dense"][0] and out["dense"][1] and out["hi"][0] == out["hi"][1]
                    and out["n_cand"][0] == n_win)
    return out


def tree_sum_addends(recs: np.ndarray, window: int) -> List[np.ndarray]:
    """The seven per-row addends of the window's time sums (model.py:241-271 expression order):
    dataloader, forward, backward, optimizer, wall, traced, dataloader + traced over usable window rows."""
    from oracle import fast_oracle

    t_start = max(0, len(recs) - int(window))
    w = recs[t_start:]
    rows = fast_oracle.window_rows(w)
    usable = (w["dur_ns"][:, USABLE_COLS] > 0).any(axis=1)
    rows = rows[usable]
    dl, f, b, o, wall = rows[:, 0], rows[:, 2], rows[:, 3], rows[:, 4], rows[:, 5]
    traced = np.maximum(wall, (f + b) + o)
    return [dl, f, b, o, wall, traced, dl + traced]


# ----------------------------------------------------------------------------- K4 / K7d inputs
K4_SIZES = (1000, 1)   # steps; neither is a multiple of K4's 64-step tile


def rank_rows(R: int, n: int, seed: int) -> np.ndarray:
    """[R, n, 8] aligned WindowRows as the pipeline produces them (ns -> ms of integer durations,
    f64 of u64 byte counts, some above 2^53): exact ties across ranks, an identical rank, all-zero
    compute (wait = wall) and walls above and below compute, lognormal durations over ~12 decades."""
    from oracle import fast_oracle

    rng = np.random.default_rng(seed)
    rec = np.zeros((R, n), dtype=STEP_RECORD_DTYPE)
    dur = np.floor(np.exp(rng.normal(np.log(1e6), 4.6, size=(R, n, 6)))).astype(np.uint64)
    tie = rng.random(n) < 0.15                       # every rank reports the same value for the step
    dur[:, tie, :] = dur[0, tie, :]
    half = rng.random(n) < 0.15                      # ranks 0 .. R/2 tie
    dur[: max(1, R // 2), half, :] = dur[0, half, :]
    zero = rng.random((R, n)) < 0.05
    dur[zero, 0] = 0
    zc = rng.random((R, n)) < 0.05
    dur[zc, 2:5] = 0
    comp = dur[:, :, 2] + dur[:, :, 3] + dur[:, :, 4]
    below = (comp.astype(np.float64) * rng.uniform(0.1, 1.0, (R, n))).astype(np.uint64)
    above = comp + np.floor(np.exp(rng.normal(np.log(1e5), 3.0, (R, n)))).astype(np.uint64)
    dur[:, :, 5] = np.where(rng.random((R, n)) < 0.5, below, above)
    idle = rng.random((R, n)) < 0.03                 # nothing at all: every column 0
    dur[idle] = 0
    rec["dur_ns"] = dur
    big = rng.random((R, n)) < 0.2
    alloc = np.where(big, rng.integers(1 << 53, 1 << 62, (R, n), dtype=np.uint64),
                     rng.integers(0, 1 << 40, (R, n), dtype=np.uint64))
    alloc[:, tie] = alloc[0, tie]
    rec["peak_alloc"] = alloc
    rec["peak_resv"] = alloc + rng.integers(0, 1 << 36, (R, n), dtype=np.uint64)
    if R >= 3:                                       # one rank identical to another
        rec[R - 1] = rec[1]
    return np.stack([fast_oracle.window_rows(rec[r]) for r in range(R)])


COMB_COLS = ((0, 6), (2, 3), (6, 2))   # (first_col, n_cols) of the K7d calls


def comb_expected(rows: np.ndarray, first_col: int, n_cols: int) -> np.ndarray:
    """[n_cols, 3, n]: per step, the median / worst / sum of the 1-D rank array, as
    live_oracle.py computes them (np.median, np.max, np.sum)."""
    R, n, _ = rows.shape
    out = np.empty((n_cols, 3, n), dtype=np.float64)
    for m in range(n_cols):
        per_step = np.ascontiguousarray(rows[:, :, first_col + m].T)   # [n, R]: one contiguous rank array per step
        out[m, 0] = np.median(per_step, axis=1)
        out[m, 1] = np.max(per_step, axis=1)
        out[m, 2] = np.sum(per_step, axis=1)   # the CPU tests pin this to np.sum of each 1-D rank array
    return out
