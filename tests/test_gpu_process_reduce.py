"""GPU: the Process section's reduce against oracle/process_oracle.py, with ``==`` on every float.

- K6 alone (k_proc_reduce -> k_finalize + k_finalize_dd): every per-rank field at the CTA, warp,
  finalize-fold (> 32 CTAs) and grid-stride (> 4 x 132 CTAs on an H100 SXM) edges, over a ring
  whose seam falls inside a warp and a CTA, and for every ``max_rows`` against what the ring
  retains;
- row families: GPU metrics on some rows only, ``used == 0`` rows (out of the overhang ratio), no
  GPU rows, cores changing inside the window, CPU readings the compensated average is sensitive
  to, byte columns whose totals pass 2^53 (a double sum rounds there; the engine's is exact);
- state: repeated launches, a small launch after a large one, K5 commits across a ring wrap;
- the whole section (``SummaryEngine.build``) for 1 to 11 ranks, an empty rank, tied peaks, the
  8-rank pooled total past 2^53, and the single-rank chained bulk build, native and Python
  drivers.

The seeds of the > 2^53 cases are ones where a double tree sum in K6's order rounds differently
from the exact sum, so a double accumulator anywhere on the path fails them.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import process_cases as pc  # noqa: E402
import replay  # noqa: E402
from helpers import oracle_proc_rows, plain  # noqa: E402

pytestmark = pytest.mark.gpu

RAM_TOTAL = replay.PROC_RAM_TOTAL_BYTES  # what oracle_proc_rows gives every row


@pytest.fixture(scope="module")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _engine(slots, rank=0, world=1):
    from traceml_b200.engine import Engine

    return Engine(device=0, rank=rank, world=world, ring_slots=64, proc_slots=int(slots))


def _load(eng, recs):
    import torch

    eng.load_procs(recs)
    torch.cuda.synchronize()


def _k6(eng, max_rows):
    import torch

    s = torch.cuda.Stream()
    l0 = eng.launch_count
    eng.proc_reduce_launch(int(max_rows), int(s.cuda_stream))
    agg = eng.proc_reduce_collect()
    return agg, eng.launch_count - l0


def _assert_k6_equals_oracle(agg, recs, where=""):
    """``recs``: exactly the rows K6 reduced (the retained, latest ``max_rows``)."""
    from oracle import process_oracle
    from traceml_b200 import sections

    n = len(recs)
    sec = process_oracle.load_section(oracle_proc_rows({0: recs}, 1), max_rows=max(1, n))
    ag, pr = sec["aggregate"], sec["per_global_rank"][0]
    has = (recs["flags"] & pc.METRICS) != 0
    n_gpu = int(has.sum())
    assert agg.n == ag["process_samples"] == n, where
    assert agg.ts_min == ag["first_ts"] and agg.ts_max == ag["last_ts"], where
    assert (agg.sum_cpu + agg.sum_cpu_lo) / n == pr["cpu_avg_percent"], (where, agg.sum_cpu, agg.sum_cpu_lo)
    assert agg.max_cpu == pr["cpu_peak_percent"], where
    # the byte sums are the exact integer sums; the averages then round once, as the reference's
    assert agg.sum_rss == sum(int(x) for x in recs["rss"]), where
    assert float(agg.sum_rss) / n == pr["ram_avg_bytes"] and agg.max_rss == pr["ram_peak_bytes"], where
    assert agg.n_gpu == n_gpu, where
    assert agg.sum_used == sum(int(x) for x in recs["mem_alloc"][has]), where
    assert agg.sum_resv == sum(int(x) for x in recs["mem_resv"][has]), where
    if n_gpu:
        assert float(agg.sum_used) / n_gpu == pr["gpu_mem_used_avg_bytes"], where
        assert float(agg.sum_resv) / n_gpu == pr["gpu_mem_reserved_avg_bytes"], where
        assert agg.max_used == pr["gpu_mem_used_peak_bytes"], where
        assert agg.max_resv == pr["gpu_mem_reserved_peak_bytes"], where
        assert agg.max_total == pr["gpu_mem_total_bytes"], where
    else:
        assert pr["gpu_mem_used_avg_bytes"] is None and pr["gpu_mem_total_bytes"] is None, where
        assert agg.max_used == agg.max_resv == agg.max_total == 0.0, where
    ratio = pr["gpu_mem_reserved_overhang_ratio"]
    assert agg.max_ratio == (-1.0 if ratio is None else ratio), (where, agg.max_ratio, ratio)
    assert agg.max_cores == pr["cpu_logical_core_count"], where
    assert bool(agg.any_gpu_available) == pr["gpu_available"], where
    # the same aggregates through the rule engine's per-rank rows (gpu_count, ram_total, averages)
    got = plain(sections.build_process({0: sections.proc_agg_dict(agg, ram_total=RAM_TOTAL, gpu_count=1)}))
    assert got["per_global_rank"]["0"] == plain(pr), where
    assert got["aggregate"] == plain(ag), where


# ----------------------------------------------------------------------------- (a) K6 alone
# 256 threads per CTA; k_finalize_dd's 32 lanes fold more than one CTA each above 32 CTAs
# (8192 rows); 135168 = 4 x 132 SMs x 256 is the grid cap on an H100 SXM, above it the
# grid-stride loop takes a second trip.
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 8192, 8193, 135_168, 135_169])
def test_k6_equals_oracle_at_grid_edges(cuda, n):
    recs = pc.make("mixed_metrics", n, seed=n)
    eng = _engine(n + 8)
    try:
        _load(eng, recs)
        agg, launches = _k6(eng, n)
        assert launches == 3
        _assert_k6_equals_oracle(agg, recs, f"n={n}")
    finally:
        eng.close()


# (slots, rows loaded, max_rows): retained = min(loaded, slots); K6 reduces the latest
# min(retained, max_rows).  1000 slots after 2500 rows: the latest 500 rows sit in slots 0-499, so
# a window of more than 500 rows crosses the seam -- at full retention 500 rows in: CTA 1, warp 7,
# lane 20.  15000 slots (1.5 x the default window) after 35013 rows, the default 10^4 rows: the
# seam is 4987 rows in -- CTA 19, warp 3, lane 27.
WRAPS = [(1000, 2500, m) for m in (1, 255, 999, 1000, 5000)] + [(15_000, 35_013, 10_000)]


@pytest.mark.parametrize("slots,loaded,max_rows", WRAPS)
def test_k6_equals_oracle_over_a_wrapped_ring(cuda, slots, loaded, max_rows):
    recs = pc.make("mixed_metrics", loaded, seed=slots + max_rows)
    eng = _engine(slots)
    try:
        _load(eng, recs)
        keep = min(loaded, slots, max_rows)
        agg, _ = _k6(eng, max_rows)
        _assert_k6_equals_oracle(agg, recs[loaded - keep:], f"slots={slots} max_rows={max_rows}")
    finally:
        eng.close()


# ----------------------------------------------------------------------------- (b) row families
FAMILY_CASES = [(f, n, 7) for f in pc.FAMILIES for n in (200, 10_001)] + [
    ("bytes_170g", 100_000, 12),   # one rank, 10^5 samples of ~170 GiB
    ("bytes_1t8", 140_000, 12),    # one rank, 1.4 x 10^5 samples of ~1.8 TiB (two grid-stride trips)
    ("bytes_1t8", 10_001, 12),
]


@pytest.mark.parametrize("family,n,seed", FAMILY_CASES)
def test_k6_equals_oracle_for_row_families(cuda, family, n, seed):
    recs = pc.make(family, n, seed=seed)
    eng = _engine(n + 8)
    try:
        _load(eng, recs)
        agg, _ = _k6(eng, n)
        _assert_k6_equals_oracle(agg, recs, f"{family} n={n}")
        if family == "all_used_zero":
            assert agg.n_gpu == n and agg.max_ratio == -1.0
        if seed == 12:  # the > 2^53 inputs
            assert agg.sum_rss > 2 ** 53 and agg.sum_used > 2 ** 53
    finally:
        eng.close()


# ----------------------------------------------------------------------------- (c) state
def test_k6_two_launches_give_identical_bytes(cuda):
    recs = pc.make("mixed_metrics", 10_001, seed=3)
    eng = _engine(10_001)
    try:
        _load(eng, recs)
        a, _ = _k6(eng, 10_000)
        b, _ = _k6(eng, 10_000)
        assert bytes(a) == bytes(b)
    finally:
        eng.close()


def test_k6_small_launch_after_a_large_one_equals_a_fresh_engine(cuda):
    n = 135_169
    recs = pc.make("bytes_1t8", n, seed=5)
    used, fresh = _engine(n), _engine(n)
    try:
        _load(used, recs)
        _load(fresh, recs)
        big, _ = _k6(used, n)  # 528 CTAs of partials left behind
        _assert_k6_equals_oracle(big, recs, "large")
        small, _ = _k6(used, 300)
        want, _ = _k6(fresh, 300)
        assert bytes(small) == bytes(want)
        _assert_k6_equals_oracle(small, recs[-300:], "small after large")
    finally:
        used.close()
        fresh.close()


def test_k5_commits_across_a_wrap_equal_the_bulk_load(cuda):
    import torch

    recs = pc.make("mixed_metrics", 150, seed=9)
    committed, loaded = _engine(64), _engine(64)
    try:
        s = torch.cuda.Stream()
        for r in recs:  # k_proc_commit, one sample per launch, wraps the 64-slot ring twice
            committed.proc_commit(int(r["seq"]), float(r["ts"]), float(r["cpu_pct"]), int(r["rss"]),
                                  int(r["mem_alloc"]), int(r["mem_resv"]), int(r["mem_total"]),
                                  int(r["flags"]), int(r["cpu_cores"]), int(s.cuda_stream))
        s.synchronize()
        _load(loaded, recs)
        for rows in (64, 40):
            a, _ = _k6(committed, rows)
            b, _ = _k6(loaded, rows)
            assert bytes(a) == bytes(b), rows
            _assert_k6_equals_oracle(a, recs[-rows:], f"commits rows={rows}")
    finally:
        committed.close()
        loaded.close()


# ----------------------------------------------------------------------------- (d) the section
def _assert_section_equals_oracle(got, procs, R, proc_rows, where=""):
    from oracle import process_oracle

    want = process_oracle.process_section(oracle_proc_rows(procs, R), max_rows=proc_rows)
    got = plain(got)
    assert got["aggregate"] == plain(want["data"]["aggregate"]), where
    assert got["per_global_rank"] == plain(want["data"]["per_global_rank"]), where
    # the rule engine's signals use the oracle's operations (max(0, a / b) * 100, first strict max,
    # (max - min) / max): scores, evidence and the formatted summaries compare exactly
    assert got["primary"] == plain(want["diagnosis"]["primary"]), where
    assert got["issues"] == plain(want["diagnosis"]["issues"]), where
    return want


def _build(procs, R, proc_rows, *, native=True, steps=None, window=100):
    import torch

    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    engines = []
    try:
        for r in range(R):
            n = len(procs[r])
            e = Engine(device=0, rank=r, world=R, ring_slots=(len(steps) + 8) if steps is not None else 64,
                       proc_slots=max(64, n + 8))
            engines.append(e)
            if steps is not None:
                e.load_steps(steps)
            if n:
                e.load_procs(procs[r])
        torch.cuda.synchronize()
        res = sections.SummaryEngine(engines, ram_total=RAM_TOTAL, gpu_count=R, native=native).build(window, proc_rows)
        return plain(res["process"]), res
    finally:
        for e in engines:
            e.close()


def _ranks_with_ties(R, seed):
    """Different sample counts per rank, rank 1 (R > 1) empty, and the first and the last non-empty
    rank tied on the RSS and the reserved peak (the first strict max must pick the lower rank)."""
    procs = {}
    for r in range(R):
        n = 0 if (R > 1 and r == 1) else 37 + 911 * r
        procs[r] = pc.make("mixed_metrics", n, seed=seed, rank=r)
    tied = [r for r in range(R) if len(procs[r])]
    tied = [tied[0], tied[-1]] if len(tied) > 1 else tied
    for r in tied:
        p, i = procs[r], len(procs[r]) // 2
        p["rss"][i], p["mem_alloc"][i], p["mem_resv"][i] = 10 * pc.GIB, 40 * pc.GIB, 60 * pc.GIB
        p["flags"][i] = pc.AVAIL | pc.METRICS
    return procs


@pytest.mark.parametrize("R", [1, 2, 3, 8, 11])
def test_process_section_equals_oracle_across_ranks(cuda, R):
    procs = _ranks_with_ties(R, seed=R)
    got, _ = _build(procs, R, 10_000)
    want = _assert_section_equals_oracle(got, procs, R, 10_000, f"R={R}")
    if R > 1:
        from oracle import process_oracle

        sig = process_oracle.signals(want["data"])
        assert sig["highest_rss_rank"] == sig["highest_reserved_rank"] == 0
        assert "1" not in got["per_global_rank"]


def test_process_section_pooled_bytes_past_2_53(cuda):
    # 8 ranks x 10^4 samples of ~170 GiB: each rank's sums are below 2^53, the pooled ones are not
    R = 8
    procs = {r: pc.make("bytes_170g", 10_000, seed=39, rank=r) for r in range(R)}
    got, _ = _build(procs, R, 10_000)
    _assert_section_equals_oracle(got, procs, R, 10_000, "pooled")
    assert sum(int(p["rss"].sum(dtype=np.uint64)) for p in procs.values()) > 2 ** 53


def test_process_section_chained_bulk_build(cuda):
    """One rank, a window above 2^17 steps: the single-rank chained build runs K6 on its side
    stream.  The native and the Python driver both equal the oracle."""
    import replay

    W = 140_000
    steps = replay.make_step_replay("balanced", 1, W, seed=21)[0]
    procs = {0: pc.make("bytes_1t8", 10_001, seed=12)}
    native, res = _build(procs, 1, 10_000, steps=steps, window=W)
    assert res["reduce"].fused_rows
    _assert_section_equals_oracle(native, procs, 1, 10_000, "native")
    python, _ = _build(procs, 1, 10_000, steps=steps, window=W, native=False)
    _assert_section_equals_oracle(python, procs, 1, 10_000, "python driver")
