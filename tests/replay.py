"""Seeded synthetic telemetry (the replay sets of SURVEY.md section 8(d)).

Produces per-rank arrays of StepRecord / ProcRecord with integer-nanosecond
durations and integer byte counts, so the CUDA path, the oracle and the
reference (through its own SQLite projection writers) all see *identical*
inputs.  Used by tests, bench.py and tests/golden/make_golden.py.

Base shape (SURVEY 8d, config 3 "input_straggler_ddp_demo" replay):
forward N(10, 0.3) ms, backward N(20, 0.3), optimizer N(3, 0.1), h2d 0.2,
dataloader 3 + U(0, 1), step wall 38 + U(0, 1); memory 4 GiB + rank * 1 MiB.
"""

from __future__ import annotations

import hashlib
from typing import Dict, Optional

import numpy as np

from traceml_b200.records import (
    FLAG_HAS_MEM,
    PHASE_BACKWARD,
    PHASE_DATALOADER,
    PHASE_FORWARD,
    PHASE_H2D,
    PHASE_OPTIMIZER,
    PHASE_STEP,
    PROC_FLAG_GPU_AVAILABLE,
    PROC_FLAG_HAS_GPU_METRICS,
    PROC_RECORD_DTYPE,
    STEP_RECORD_DTYPE,
)

GIB = 1024 ** 3
MIB = 1024 ** 2
GPU_TOTAL_BYTES = 183_359 * MIB  # a synthetic device total; the golden vectors were made with it

STEP_SCENARIOS = (
    "balanced", "input_straggler", "compute_straggler", "straggler",
    "input_bound", "wait_heavy", "compute_bound", "warmup", "ragged",
    "trend_worsening", "duplicates", "empty_rank", "no_overlap",
    "mem_creep_confirmed", "mem_creep_early", "mem_imbalance", "mem_pressure",
    "cpu_only",
)

PROC_SCENARIOS = (
    "normal", "very_high_gpu", "high_gpu", "overhang", "imbalance",
    "high_rss", "high_cpu", "no_gpu",
)


def _ms_to_ns(ms: np.ndarray) -> np.ndarray:
    return np.maximum(np.rint(np.asarray(ms, dtype=np.float64) * 1.0e6), 0).astype(np.uint64)


def make_step_replay(
    scenario: str,
    n_ranks: int,
    n_steps: int,
    seed: int = 0,
    first_step: int = 1,
    only_ranks=None,
) -> Dict[int, np.ndarray]:
    """Return ``{rank: StepRecord[n]}`` for one named scenario (``only_ranks``
    restricts generation to some ranks of the same n_ranks-wide job)."""
    if scenario not in STEP_SCENARIOS:
        raise ValueError(f"unknown step scenario {scenario!r}")
    out: Dict[int, np.ndarray] = {}
    for rank in (range(n_ranks) if only_ranks is None else only_ranks):
        rng = np.random.default_rng([int(seed), int(rank), 0xB200])
        n = int(n_steps)
        if scenario == "warmup":
            n = min(n, 40)
        steps = np.arange(first_step, first_step + n, dtype=np.uint64)
        t = np.linspace(0.0, 1.0, n) if n > 1 else np.zeros(n)

        fwd = rng.normal(10.0, 0.3, n)
        bwd = rng.normal(20.0, 0.3, n)
        opt = rng.normal(3.0, 0.1, n)
        h2d = np.full(n, 0.2)
        dl = 3.0 + rng.uniform(0.0, 1.0, n)
        wall = 38.0 + rng.uniform(0.0, 1.0, n)
        alloc = np.full(n, 4 * GIB + rank * MIB, dtype=np.float64) + rng.integers(0, 4096, n)
        resv = alloc + 256 * MIB

        if scenario in ("input_straggler", "straggler") and rank == 0:
            dl = 250.0 + rng.uniform(0.0, 1.0, n)
        if scenario in ("compute_straggler", "straggler") and rank == (1 % n_ranks):
            bwd = bwd * 1.5
            wall = wall + 10.0
        if scenario == "input_bound":
            dl = 20.0 + rng.uniform(0.0, 1.0, n)
        if scenario == "wait_heavy":
            wall = 50.0 + rng.uniform(0.0, 1.0, n)
        if scenario == "compute_bound":
            wall = 33.5 + rng.uniform(0.0, 0.2, n)
        if scenario == "trend_worsening":
            dl = (20.0 + rng.uniform(0.0, 1.0, n)) * (1.0 + 0.6 * t)
        if scenario == "ragged":
            steps = steps + np.uint64(7 * rank)
        if scenario == "no_overlap":
            steps = steps + np.uint64((n + 5) * rank)
        if scenario == "mem_creep_confirmed":
            alloc = alloc + 2.0 * GIB * t
            resv = resv + 2.0 * GIB * t
        if scenario == "mem_creep_early":
            alloc = alloc + 0.1 * GIB * t
            resv = resv + 0.1 * GIB * t
        if scenario == "mem_imbalance" and rank == (2 % n_ranks):
            alloc = alloc * 1.25
            resv = resv * 1.25
        if scenario == "mem_pressure":
            resv = np.full(n, 0.95 * GPU_TOTAL_BYTES) + rank * MIB

        rec = np.zeros(n, dtype=STEP_RECORD_DTYPE)
        rec["step"] = steps
        rec["dur_ns"][:, PHASE_DATALOADER] = _ms_to_ns(dl)
        rec["dur_ns"][:, PHASE_H2D] = _ms_to_ns(h2d)
        rec["dur_ns"][:, PHASE_FORWARD] = _ms_to_ns(fwd)
        rec["dur_ns"][:, PHASE_BACKWARD] = _ms_to_ns(bwd)
        rec["dur_ns"][:, PHASE_OPTIMIZER] = _ms_to_ns(opt)
        rec["dur_ns"][:, PHASE_STEP] = _ms_to_ns(wall)
        rec["n_calls"][:] = 1
        rec["peak_alloc"] = np.rint(alloc).astype(np.uint64)
        rec["peak_resv"] = np.rint(resv).astype(np.uint64)
        rec["host_ts"] = 1.7e9 + np.cumsum(np.asarray(wall) + np.asarray(dl)) / 1000.0
        gpu_mask = (1 << PHASE_H2D) | (1 << PHASE_FORWARD) | (1 << PHASE_BACKWARD) | (1 << PHASE_OPTIMIZER)
        rec["gpu_mask"] = gpu_mask
        rec["flags"] = FLAG_HAS_MEM
        if scenario == "cpu_only":
            rec["gpu_mask"] = 0
            rec["flags"] = 0
            rec["peak_alloc"] = 0
            rec["peak_resv"] = 0
            rec["n_calls"][:, PHASE_H2D] = 0
            rec["dur_ns"][:, PHASE_H2D] = 0

        if scenario == "ragged" and rank == (1 % n_ranks) and n > 12:
            rec = np.delete(rec, [n // 2, n // 2 + 3])  # holes in one rank
        if scenario == "duplicates" and n > 20:
            # a failed step flushes again under the old id (sdk/instrumentation.py:188-198)
            dup = rec[[n // 3, 2 * n // 3]].copy()
            dup["dur_ns"][:, PHASE_FORWARD] += np.uint64(5_000_000)
            dup["peak_alloc"] += np.uint64(123 * MIB)
            rec = np.concatenate([rec[: n // 3 + 1], dup[:1], rec[n // 3 + 1: 2 * n // 3 + 1],
                                  dup[1:], rec[2 * n // 3 + 1:]])
        if scenario == "empty_rank" and rank == n_ranks - 1 and n_ranks > 1:
            rec = rec[:0]
        rec["seq"] = np.arange(len(rec), dtype=np.uint64)
        out[rank] = rec
    return out


def make_proc_replay(
    scenario: str,
    n_ranks: int,
    n_samples: int,
    seed: int = 0,
    period_s: float = 0.001,
    only_ranks=None,
) -> Dict[int, np.ndarray]:
    """Return ``{rank: ProcRecord[n]}`` (1 kHz by default -- BASELINE config 4)."""
    if scenario not in PROC_SCENARIOS:
        raise ValueError(f"unknown process scenario {scenario!r}")
    out: Dict[int, np.ndarray] = {}
    for rank in (range(n_ranks) if only_ranks is None else only_ranks):
        rng = np.random.default_rng([int(seed), int(rank), 0x9C])
        n = int(n_samples)
        rec = np.zeros(n, dtype=PROC_RECORD_DTYPE)
        rec["seq"] = np.arange(1, n + 1, dtype=np.uint64)
        rec["ts"] = 1.7e9 + period_s * np.arange(n) + 1e-5 * rank
        cpu = 95.0 + rng.normal(0.0, 5.0, n)
        rss = 6 * GIB + rng.integers(0, 64 * MIB, n)
        used = 40 * GIB + rank * 64 * MIB + rng.integers(0, 16 * MIB, n)
        resv = used + 4 * GIB
        if scenario == "very_high_gpu":
            resv = np.full(n, int(0.93 * GPU_TOTAL_BYTES)) + rank * MIB
        if scenario == "high_gpu":
            resv = np.full(n, int(0.84 * GPU_TOTAL_BYTES)) + rank * MIB
        if scenario == "overhang" and rank == (1 % n_ranks):
            resv = (used * 1.8).astype(np.int64)
        if scenario == "imbalance" and rank == 0:
            used = used // 3
            resv = used + 1 * GIB
        if scenario == "high_rss":
            rss = np.full(n, 440 * GIB) + rng.integers(0, MIB, n)
        if scenario == "high_cpu":
            cpu = 900.0 + rng.normal(0.0, 5.0, n)
        rec["cpu_pct"] = np.maximum(cpu, 0.0)
        rec["rss"] = rss.astype(np.uint64)
        rec["cpu_cores"] = 8 if scenario == "high_cpu" else 192
        if scenario == "no_gpu":
            rec["flags"] = 0
        else:
            rec["mem_alloc"] = np.asarray(used).astype(np.uint64)
            rec["mem_resv"] = np.asarray(resv).astype(np.uint64)
            rec["mem_total"] = GPU_TOTAL_BYTES
            rec["flags"] = PROC_FLAG_GPU_AVAILABLE | PROC_FLAG_HAS_GPU_METRICS
        out[rank] = rec
    return out


PROC_RAM_TOTAL_BYTES = float(512 * GIB)


def replay_digest(records_by_rank: Dict[int, np.ndarray]) -> str:
    """sha256 over the raw record bytes: pins the generator in golden files."""
    h = hashlib.sha256()
    for rank in sorted(records_by_rank):
        h.update(int(rank).to_bytes(4, "little"))
        h.update(np.ascontiguousarray(records_by_rank[rank]).tobytes())
    return h.hexdigest()


__all__ = [
    "STEP_SCENARIOS", "PROC_SCENARIOS", "GPU_TOTAL_BYTES", "PROC_RAM_TOTAL_BYTES",
    "make_step_replay", "make_proc_replay", "replay_digest",
]
