#!/usr/bin/env python
"""The UNMODIFIED reference (traceopt-ai/traceml 0.2.15, installed into the git-ignored
``oracle/_ref`` by ``oracle/install_reference.py``) timed on the host's cores.

This file never imports the engine (``traceml_b200.engine`` / ``_abi`` / any ``.so`` of this
repository): ``bench.py --impl reference`` runs it as a separate process so that the
reference-arm process maps none of the repository's native code.  The only thing shared with the
product arm is the seeded synthetic generator (``tests/replay.py``) and the pure-Python record
description (``traceml_b200/records.py``), so both arms reduce IDENTICAL inputs.

legs
  reduce    R ranks x ROWS step records (+ process samples) are projected into a SQLite file by the
            reference's own writers (``aggregator/sqlite_writers/*.build_rows/insert_rows``), then
            ``StepTimeSummarySection(max_rows=W).build(db)``, ``StepMemorySummarySection(
            window_size=W).build(db)`` and ``ProcessSummarySection().build(db)`` are timed
            (SURVEY 8d(ii)); single-threaded Python, as the reference runs it.
  overhead  per-step wall of a training loop untraced vs inside the reference's real
            ``traceml.trace_step`` (auto mode: patches, CUDA-event timers, StepMemoryTracker),
            with ``StepTimeSampler.sample()`` / ``StepMemorySampler.sample()`` every 64 steps as
            the sampler thread's amortised share (SURVEY 8d(i)).

Prints ONE JSON object on the last line of stdout.
"""
from __future__ import annotations

import argparse
import json
import os
import sqlite3
import statistics
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")


def _paths():
    if not os.path.isdir(os.path.join(REF, "traceml")):
        raise SystemExit(json.dumps({"unavailable": f"{REF} holds no installed reference"}))
    sys.path.insert(0, REF)
    sys.path.insert(1, ROOT)
    sys.path.insert(2, os.path.join(ROOT, "tests"))
    os.environ.setdefault("TRACEML_LOGS_DIR", tempfile.mkdtemp(prefix="traceml_ref_logs_"))


def _envelope(sampler, rank, world, rows):
    return {"rank": rank, "global_rank": rank, "local_rank": rank, "world_size": world,
            "local_world_size": world, "node_rank": 0, "hostname": "bench-host", "pid": 1000 + rank,
            "sampler": sampler, "timestamp": 0.0, "tables": {"t": rows}}


def build_db(path, step_records, proc_records, ram_total):
    """Replay records -> the reference's SQLite projection tables, through its own writers
    (aggregator/sqlite_writers/step_time.py:172-187, step_memory.py:139-156, process.py:169-190)."""
    from traceml.aggregator.sqlite_writers import process as proc_w
    from traceml.aggregator.sqlite_writers import step_memory as mem_w
    from traceml.aggregator.sqlite_writers import step_time as time_w
    from traceml_b200 import records as rec_mod  # pure-Python record description, no native code

    conn = sqlite3.connect(path)
    time_w.init_schema(conn); mem_w.init_schema(conn); proc_w.init_schema(conn)
    recv, world = 1, len(step_records)
    t0 = time.perf_counter()
    n_rows = 0
    for rank in sorted(step_records):
        recs = step_records[rank]
        trows = [rec_mod.step_record_to_wire(r, device=f"cuda:{rank}") for r in recs]
        mrows = [rec_mod.step_record_to_memory_wire(r, device=f"cuda:{rank}") for r in recs]
        time_w.insert_rows(conn, time_w.build_rows(_envelope("StepTimeSampler", rank, world, trows), recv))
        mem_w.insert_rows(conn, mem_w.build_rows(_envelope("StepMemorySampler", rank, world, mrows), recv))
        n_rows += 2 * len(recs)
        recv += 1
    for rank in sorted(proc_records or {}):
        rows = [rec_mod.proc_record_to_wire(r, pid=1000 + rank, ram_total=ram_total, gpu_count=world,
                                            device_index=rank) for r in proc_records[rank]]
        proc_w.insert_rows(conn, proc_w.build_rows(_envelope("ProcessSampler", rank, world, rows), recv))
        n_rows += len(rows)
        recv += 1
    conn.commit(); conn.close()
    return n_rows, time.perf_counter() - t0


def leg_reduce(args):
    import replay
    from traceml.reporting.sections.process import ProcessSummarySection
    from traceml.reporting.sections.step_memory import StepMemorySummarySection
    from traceml.reporting.sections.step_time import StepTimeSummarySection

    R, rows, W = args.ranks, args.rows, args.window or args.rows
    recs = replay.make_step_replay(args.scenario, R, rows, seed=args.seed)
    procs = replay.make_proc_replay("normal", R, args.proc_rows, seed=args.seed)
    td = tempfile.mkdtemp(prefix="traceml_ref_db_")
    db = os.path.join(td, "telemetry.sqlite")
    n_ins, t_ins = build_db(db, recs, procs, replay.PROC_RAM_TOTAL_BYTES)

    def once():
        t0 = time.perf_counter()
        st = StepTimeSummarySection(max_rows=W).build(db)
        t1 = time.perf_counter()
        sm = StepMemorySummarySection(window_size=W).build(db)
        t2 = time.perf_counter()
        pr = ProcessSummarySection().build(db)
        t3 = time.perf_counter()
        return (t3 - t0, t1 - t0, t2 - t1, t3 - t2), (st, sm, pr)

    for _ in range(args.warmup):
        once()
    times, last = [], None
    for _ in range(args.steps):
        t, last = once()
        times.append(t)
    st, sm, pr = last
    diag = {}
    for name, res in (("step_time", st), ("step_memory", sm), ("process", pr)):
        p = getattr(res, "payload", None) or {}
        d = (p.get("diagnosis") or {}) if isinstance(p, dict) else {}
        g = (p.get("global") or {}) if isinstance(p, dict) else {}
        diag[name] = {"status": d.get("status"), "reason": d.get("reason"),
                      "global": {k: g.get(k) for k in ("average", "median", "worst") if k in g},
                      "metadata": {k: v for k, v in (p.get("metadata") or {}).items()
                                   if isinstance(v, (int, float, str, type(None)))}}
    out = {
        "leg": "reduce", "ranks": R, "rows_per_rank": rows, "window": W, "scenario": args.scenario,
        "seed": args.seed, "steps": len(times), "warmup": args.warmup,
        "s_per_step": [t[0] for t in times],
        "s_per_step_median": statistics.median(t[0] for t in times),
        "s_sections_median": {"step_time": statistics.median(t[1] for t in times),
                              "step_memory": statistics.median(t[2] for t in times),
                              "process": statistics.median(t[3] for t in times)},
        "us_per_row": statistics.median(t[0] for t in times) / (R * rows) * 1e6,
        "sqlite_projection": {"rows": n_ins, "s": t_ins, "us_per_row": t_ins / max(1, n_ins) * 1e6},
        "summary": diag,
        "cores_used": 1, "host_cores": os.cpu_count(),
        "reference_version": _ref_version(),
    }
    print(json.dumps(out))


def _ref_version():
    try:
        import traceml

        return {"file": os.path.relpath(traceml.__file__, ROOT), "version": getattr(traceml, "__version__", None)}
    except Exception as exc:  # pragma: no cover
        return {"error": str(exc)}


# ----------------------------------------------------------------------------- overhead
def resnet18(num_classes=10):
    import torch
    import torch.nn as nn

    class Block(nn.Module):
        def __init__(self, cin, cout, stride):
            super().__init__()
            self.c1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False); self.b1 = nn.BatchNorm2d(cout)
            self.c2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False); self.b2 = nn.BatchNorm2d(cout)
            self.down = None
            if stride != 1 or cin != cout:
                self.down = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.BatchNorm2d(cout))

        def forward(self, x):
            y = torch.relu(self.b1(self.c1(x)))
            y = self.b2(self.c2(y))
            return torch.relu(y + (x if self.down is None else self.down(x)))

    layers = [nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(), nn.MaxPool2d(3, 2, 1)]
    cin = 64
    for cout, stride in ((64, 1), (64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1)):
        layers.append(Block(cin, cout, stride)); cin = cout
    layers += [nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(512, num_classes)]
    return nn.Sequential(*layers)


def leg_overhead(args):
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"leg": "overhead", "unavailable": "no CUDA device"}))
        return
    import traceml
    from traceml.samplers.step_memory_sampler import StepMemorySampler
    from traceml.samplers.step_time_sampler import StepTimeSampler

    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    traceml.init(mode="auto")
    ts, ms = StepTimeSampler(), StepMemorySampler()
    lossf = torch.nn.functional.cross_entropy
    out = {"leg": "overhead", "reference_version": _ref_version()}

    def run_arm(traced, model, opt, xs, ys, n):
        torch.cuda.synchronize(device)
        t0 = time.perf_counter()
        for i in range(n):
            x, y = xs[i % len(xs)], ys[i % len(ys)]
            if traced:
                with traceml.trace_step(model):
                    xd, yd = x.to(device, non_blocking=True), y.to(device, non_blocking=True)
                    loss = lossf(model(xd), yd); loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)
                if i % 64 == 63:
                    ts.sample(); ms.sample()  # the sampler thread's work, amortised
            else:
                xd, yd = x.to(device, non_blocking=True), y.to(device, non_blocking=True)
                loss = lossf(model(xd), yd); loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize(device)
        if traced:
            ts.sample(); ms.sample()
        return (time.perf_counter() - t0) / n * 1.0e6

    def harness(name, model, xs, ys, n, cycles):
        opt = torch.optim.SGD(model.parameters(), lr=1e-3)
        for traced in (False, True):
            run_arm(traced, model, opt, xs, ys, max(5, n // 4))
        res = {False: [], True: []}
        for _ in range(cycles):
            for traced in (False, True):
                res[traced].append(run_arm(traced, model, opt, xs, ys, n))
        base = statistics.median(res[False])
        out[name] = {"untraced_us": base, "reference_us": statistics.median(res[True]),
                     "reference_overhead_us": statistics.median(res[True]) - base,
                     "steps_per_cycle": n, "cycles": cycles}

    torch.manual_seed(0)
    mlp = torch.nn.Linear(8, 8).to(device)
    xs = [torch.randn(16, 8).pin_memory() for _ in range(8)]
    ys = [torch.randint(0, 8, (16,)).pin_memory() for _ in range(8)]
    harness("micro_mlp", mlp, xs, ys, 100 if args.quick else 400, 3 if args.quick else 5)
    model = resnet18().to(device)
    xs = [torch.randn(64, 3, 224, 224).pin_memory() for _ in range(2)]
    ys = [torch.randint(0, 10, (64,)).pin_memory() for _ in range(2)]
    harness("resnet18_b64", model, xs, ys, 8 if args.quick else 24, 2 if args.quick else 3)
    rows = list(ts.db.get_table("StepTimeTable") or [])
    out["step_rows_recorded"] = len(rows)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--leg", required=True, choices=["reduce", "overhead"])
    ap.add_argument("--ranks", type=int, default=1)
    ap.add_argument("--rows", type=int, default=10_000)
    ap.add_argument("--window", type=int, default=0)
    ap.add_argument("--proc-rows", type=int, default=2_000)
    ap.add_argument("--scenario", default="balanced")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    _paths()
    (leg_reduce if args.leg == "reduce" else leg_overhead)(args)


if __name__ == "__main__":
    main()
