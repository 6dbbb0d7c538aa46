"""Process-sample families for the K6 (k_proc_reduce) and ``tml_diag_process`` tests.

``make(family, n, seed)`` returns ``ProcRecord[n]`` of one rank, 1 kHz timestamps.  Each family
stresses one column of the reduce: GPU-metric flags mixed inside a window, ``used == 0`` rows that
must stay out of the overhang ratio, cores that change inside the window, CPU readings the
compensated average is sensitive to, and byte columns whose totals pass 2^53 (where a double sum
stops being exact).  Rows without ``HAS_GPU_METRICS`` keep non-zero garbage in their GPU columns:
the reduce must ignore them, as the reference's loader does (it never sees them).

``replay.make_proc_replay`` is pinned by golden digests; this generator is free to change.
"""
from __future__ import annotations

import numpy as np

from traceml_b200.records import (PROC_FLAG_GPU_AVAILABLE as AVAIL, PROC_FLAG_HAS_GPU_METRICS as METRICS,
                                  PROC_RECORD_DTYPE)

MIB, GIB, TIB = 1 << 20, 1 << 30, 1 << 40

FAMILIES = ("default", "mixed_metrics", "available_no_metrics", "used_zero", "all_used_zero", "no_gpu",
            "cores_vary", "cpu_one_decimal", "cpu_zeros", "cpu_integers", "cpu_ties", "cpu_decades",
            "bytes_170g", "bytes_1t8")


def make(family: str, n: int, seed: int = 0, rank: int = 0) -> np.ndarray:
    if family not in FAMILIES:
        raise ValueError(f"unknown process family {family!r}")
    rng = np.random.default_rng([int(seed), int(rank), int(n), FAMILIES.index(family)])
    rec = np.zeros(int(n), dtype=PROC_RECORD_DTYPE)
    rec["seq"] = np.arange(1, n + 1, dtype=np.uint64)
    rec["ts"] = 1.7e9 + 1e-3 * np.arange(n) + 1e-5 * rank
    cpu = rng.uniform(0.0, 400.0, n)
    rss = 6 * GIB + rng.integers(0, 256 * MIB, n)
    used = 40 * GIB + rng.integers(0, 2 * GIB, n)
    resv = used + rng.integers(0, 8 * GIB, n)
    total = np.full(n, 80 * GIB)
    cores = np.full(n, 64)
    flags = np.full(n, AVAIL | METRICS)
    if family == "mixed_metrics":  # the sampler's rows with and without torch.cuda memory readings
        flags = np.where(rng.random(n) < 0.5, AVAIL | METRICS, AVAIL)
        total = np.where(flags & METRICS, total, 96 * GIB)  # garbage a flag-blind MAX would pick up
    elif family == "available_no_metrics":
        flags[:] = AVAIL
    elif family == "used_zero":  # used == 0 rows count in the averages but not in the ratio
        used = np.where(rng.random(n) < 0.3, 0, used)
        resv = np.where(used == 0, 70 * GIB, resv)  # would be an infinite / the largest ratio
    elif family == "all_used_zero":
        used[:] = 0
    elif family == "no_gpu":
        flags[:] = 0
    elif family == "cores_vary":
        cores = rng.integers(1, 257, n)
    elif family == "cpu_one_decimal":  # psutil's cpu_percent: one decimal
        cpu = np.round(rng.uniform(0.0, 800.0, n), 1)
    elif family == "cpu_zeros":
        cpu[:] = 0.0
    elif family == "cpu_integers":
        cpu = rng.integers(0, 1600, n).astype(np.float64)
    elif family == "cpu_ties":  # a handful of values, the peak repeated many times
        cpu = rng.choice(np.array([0.1, 12.5, 99.9, 100.0, 799.9]), n)
    elif family == "cpu_decades":  # magnitudes over 26 decades, both signs of exponent
        cpu = 10.0 ** rng.uniform(-13.0, 13.0, n)
    elif family == "bytes_170g":  # a 180 GB-class part nearly full: 10^5 rows sum past 2^53
        rss = 170 * GIB + rng.integers(0, GIB, n)
        used = 170 * GIB + rng.integers(0, GIB, n)
        resv = used + rng.integers(0, 8 * GIB, n)
        total = np.full(n, 180 * GIB)
    elif family == "bytes_1t8":  # 1.8 TiB per row: 5 * 10^3 rows already pass 2^53
        base = int(1.8 * TIB)
        rss = base + rng.integers(0, GIB, n)
        used = base + rng.integers(0, GIB, n)
        resv = used + rng.integers(0, 8 * GIB, n)
        total = np.full(n, 2 * TIB)
    rec["cpu_pct"] = cpu
    rec["rss"] = np.asarray(rss).astype(np.uint64)
    rec["mem_alloc"] = np.asarray(used).astype(np.uint64)
    rec["mem_resv"] = np.asarray(resv).astype(np.uint64)
    rec["mem_total"] = np.asarray(total).astype(np.uint64)
    rec["flags"] = flags
    rec["cpu_cores"] = cores
    return rec
