"""CPU: ``tml_diag_process`` pools per-rank byte sums exactly.

Per-rank aggregates are built here the way K6 hands them over -- exact integer byte sums, the cpu
sum as the double-double of its exact value -- from seeded integer rows whose pooled byte totals
pass 2^53.  The section's averages must equal ``process_oracle.load_section`` on the same rows with
``==``: the reference sums integers exactly and rounds once, where a double accumulator rounds at
every addition past 2^53.
"""
import os
import sys
from fractions import Fraction

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import process_cases as pc  # noqa: E402
import replay  # noqa: E402
from helpers import oracle_proc_rows, plain  # noqa: E402
from oracle import process_oracle  # noqa: E402
from traceml_b200 import _abi, sections  # noqa: E402


def _k6_agg(recs):
    """A high-precision restatement of K6 over ``recs`` (one rank, every row in the window)."""
    a = _abi.ProcAgg()
    a.n = n = len(recs)
    a.max_ratio = -1.0
    if not n:
        return a
    has = (recs["flags"] & pc.METRICS) != 0
    a.n_gpu = int(has.sum())
    a.ts_min, a.ts_max = float(recs["ts"].min()), float(recs["ts"].max())
    exact = sum(Fraction(float(x)) for x in recs["cpu_pct"])
    a.sum_cpu = float(exact)
    a.sum_cpu_lo = float(exact - Fraction(a.sum_cpu))
    a.max_cpu = float(recs["cpu_pct"].max())
    a.sum_rss, a.max_rss = sum(int(x) for x in recs["rss"]), float(recs["rss"].max())
    if a.n_gpu:
        used, resv = recs["mem_alloc"][has], recs["mem_resv"][has]
        a.sum_used, a.max_used = sum(int(x) for x in used), float(used.max())
        a.sum_resv, a.max_resv = sum(int(x) for x in resv), float(resv.max())
        a.max_total = float(recs["mem_total"][has].max())
        ratios = [float(r) / float(u) for u, r in zip(used, resv) if u > 0]
        a.max_ratio = max(ratios) if ratios else -1.0
    a.max_cores = int(recs["cpu_cores"].max())
    a.any_gpu_available = int(((recs["flags"] & pc.AVAIL) != 0).any())
    return a


# (family, ranks, rows per rank, seed): with more than one rank, each seed rounds a double pooling
# of these totals away from the exact one in at least one byte column
CASES = [
    ("bytes_170g", 8, 10_000, 39),   # per-rank sums < 2^53, the pooled 8 x 10^4 rows past it
    ("bytes_170g", 8, 10_000, 1),
    ("bytes_170g", 8, 10_000, 3),
    ("bytes_1t8", 3, 10_001, 12),    # per-rank sums already past 2^53
    ("bytes_1t8", 1, 10_001, 12),    # nothing to pool: the u64 sum rounds once, into the average
]


@pytest.mark.parametrize("family,R,n,seed", CASES)
def test_pooled_byte_averages_equal_the_oracle(family, R, n, seed):
    procs = {r: pc.make(family, n, seed=seed, rank=r) for r in range(R)}
    aggs = {r: sections.proc_agg_dict(_k6_agg(procs[r]), ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)
            for r in range(R)}
    got = plain(sections.build_process(aggs))
    want = process_oracle.process_section(oracle_proc_rows(procs, R), max_rows=n)
    assert sum(int(x) for p in procs.values() for x in p["mem_alloc"]) > 2 ** 53
    for k in ("ram_avg_bytes", "gpu_mem_used_avg_bytes", "gpu_mem_reserved_avg_bytes"):
        assert got["aggregate"][k] == want["data"]["aggregate"][k], k
    assert got["aggregate"] == plain(want["data"]["aggregate"])
    assert got["per_global_rank"] == plain(want["data"]["per_global_rank"])
    assert got["primary"] == plain(want["diagnosis"]["primary"])
    assert got["issues"] == plain(want["diagnosis"]["issues"])
