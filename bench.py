#!/usr/bin/env python
"""bench.py -- the reference's headline metric on H100.

BASELINE.json metric: "per-step profiling overhead (us) at 1/2/4/8 ranks;
cross-rank reduce GB/s".  One invocation measures both legs:

  reduce leg   (``metric``/``value``/``roofline``/``e2e``/``parity``/``default_window``)
      workload = BASELINE config 4's NVLink-reduce stress replay: every rank holds
      W step records (default W = 4e6 ~ 1 kHz x 67 min) plus 60 000 process samples.
      A "step" is one full cross-rank window reduce (align -> exchange -> per-step
      median/worst -> trend bands -> process aggregates -> rule engines).
      value = algorithmic bytes B_reduce(R, W) = R*W*64 + 128*W + 72*R per step / time,
      records resident in HBM.  e2e = same, but each step starts from HOST (pinned)
      StepRecord buffers: H2D of W*128 B per rank + reduce + results back on the host.
      parity = the W-sized result checked against the numpy oracle (oracle/fast_oracle.py,
      pinned == to the row-level oracle, pinned == to the unmodified reference) on the same
      seed, outside the timed region.  default_window = the reference's default W = 10^4 on
      the same seed in BOTH arms: this engine's time next to the UNMODIFIED reference's
      (oracle/_ref, separate process), and their summaries compared field by field.
  step leg     (``step_overhead``)
      BASELINE config 2: synthetic ResNet-18 (batch 64x3x224x224, DDP when N > 1)
      and the isolated tiny-MLP micro-harness; per-step wall of untraced vs traced
      (this engine, auto mode); the reference's real ``traceml.trace_step`` is timed by
      baseline/reference_legs.py in its own process (rank 0).

``--impl reference`` runs the UNMODIFIED reference (``oracle/_ref``, git-ignored, installed by
``oracle/install_reference.py``) in a separate process that maps none
of this repository's native code: its own SQLite projection writers + its three summary
sections on a bounded sample of the same workload (K timed steps, W warm-up; the sample per step is
sized from K so that the whole run costs ~100 s of reference time, never above --sample rows), the default-window
line at full size, and the real ``traceml.trace_step`` overhead leg.  If ``oracle/_ref`` is
missing it falls back to the oracle port and says so (``cpu_baseline.kind: "port"``).

Launch: ``python bench.py --gpus N --steps K --warmup W`` (N = 1) or under
``python -m torch.distributed.run --nproc-per-node N ... bench.py --gpus N ...``.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def b_reduce(R: int, W: int) -> float:
    """Algorithmic bytes of one window reduce (SURVEY 8d)."""
    return float(R) * W * 64.0 + 128.0 * W + 72.0 * R


def dist_setup():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return rank, local, world


def barrier(world):
    if world > 1:
        torch.distributed.barrier()


def max_over_ranks(x: float, world: int, device) -> float:
    if world <= 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=device)
    torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
    return float(t.item())


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index = index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                 "--format=csv,noheader,nounits", "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                  "sw_power_cap"), f[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None,
                "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons),
                "samples": len(sm)}


# ----------------------------------------------------------------------------- models
def resnet18(num_classes=10):
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


def step_overhead(device, world, local, quick=False):
    """Per-step wall: untraced vs this engine (auto mode).  The reference's real
    ``traceml.trace_step`` runs in its own process (baseline/reference_legs.py, rank 0)."""
    import traceml_b200 as traceml

    traceml.init(mode="auto")
    out = {}

    def run_arm(arm, model, opt, xs, ys, n):
        lossf = torch.nn.functional.cross_entropy
        torch.cuda.synchronize(device)
        t0 = time.perf_counter()
        for i in range(n):
            x, y = xs[i % len(xs)], ys[i % len(ys)]
            if arm == "untraced":
                xd, yd = x.to(device, non_blocking=True), y.to(device, non_blocking=True)
                loss = lossf(model(xd), yd); loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)
            else:
                with traceml.trace_step(model):
                    xd, yd = x.to(device, non_blocking=True), y.to(device, non_blocking=True)
                    loss = lossf(model(xd), yd); loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize(device)
        return (time.perf_counter() - t0) / n * 1.0e6

    def harness(name, model, xs, ys, n, cycles):
        opt = torch.optim.SGD(model.parameters(), lr=1e-3)
        for arm in ("untraced", "b200"):
            run_arm(arm, model, opt, xs, ys, max(5, n // 4))  # warm-up
        res = {"untraced": [], "b200": []}
        for _ in range(cycles):
            for arm in res:
                res[arm].append(run_arm(arm, model, opt, xs, ys, n))
        base = statistics.median(res["untraced"])
        out[name] = {
            "untraced_us": base,
            "b200_us": statistics.median(res["b200"]),
            "b200_overhead_us": statistics.median(res["b200"]) - base,
            "steps_per_cycle": n, "cycles": cycles,
        }

    # raw per-call host cost of the step-path entry points (tight loops, sync at the end)
    try:
        from traceml_b200 import runtime as _rt

        eng = _rt.get_engine()
        h, sp = eng._h, torch.cuda.current_stream(device).cuda_stream
        n = 3000

        def cost(fn):
            torch.cuda.synchronize(device)
            t0 = time.perf_counter()
            for _ in range(n):
                fn()
            dt = (time.perf_counter() - t0) / n * 1e6
            torch.cuda.synchronize(device)
            return dt

        ev_pool = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        out["api_cost_us"] = {
            "begin_end_pair": cost(lambda: eng._end(h, 2, eng._begin(h, 2, sp), sp)),
            "phase_host": cost(lambda: eng._host(h, 5, 1000)),
            "step_commit": cost(lambda: eng._commit(h, 1, 0, 0, 0, 0.0, sp)),
            "cuda_event_record_pair": cost(lambda: (ev_pool[0].record(), ev_pool[1].record())),
            "empty_lambda": cost(lambda: None),
        }
        eng.drain()
        # sustained telemetry rate: commit + drain (step records) and 1 kHz-style process samples
        side = torch.cuda.Stream(device=device)
        n_rec, got, t0 = 50_000, 0, time.perf_counter()
        for i in range(n_rec):
            eng._host(h, 5, 1000)
            eng._commit(h, i + 1, 0, 0, 0, 0.0, sp)
            if i % 2048 == 2047:
                got += len(eng.drain()[0])
        torch.cuda.synchronize(device)
        got += len(eng.drain()[0])
        dt = time.perf_counter() - t0
        t1 = time.perf_counter()
        pgot = 0
        for i in range(n_rec):
            eng.proc_commit(i + 1, 0.0, 50.0, 1 << 30, 1 << 30, 1 << 31, 1 << 37, 3, 64, side.cuda_stream)
            if i % 4096 == 4095:
                pgot += len(eng.proc_drain()[0])
        torch.cuda.synchronize(device)
        pgot += len(eng.proc_drain()[0])
        dt2 = time.perf_counter() - t1
        out["telemetry_rate"] = {"step_records_per_s": n_rec / dt, "step_records_drained": got,
                                 "proc_samples_per_s": n_rec / dt2, "proc_samples_drained": pgot,
                                 "records": n_rec}
        # BASELINE config 4: native sampler thread at 1 kHz for one second, GIL kept busy
        try:
            from traceml_b200.utils import timing as _tm

            if _tm._FAST is not None:
                eng.proc_drain()
                _tm._FAST.sampler_start(1000, 0)
                t2, spin = time.perf_counter(), 0
                while time.perf_counter() - t2 < 1.0:
                    spin += 1
                last, late = _tm._FAST.sampler_stop()
                el = time.perf_counter() - t2
                out["telemetry_rate"]["native_sampler"] = {
                    "requested_hz": 1000, "achieved_hz": last / el, "late_periods": late,
                    "drained": len(eng.proc_drain()[0])}
        except Exception as exc:
            out["telemetry_rate"]["native_sampler"] = {"error": str(exc)}
    except Exception as exc:
        out["api_cost_us"] = {"error": str(exc)}

    torch.manual_seed(0)
    mlp = torch.nn.Linear(8, 8).to(device)
    xs = [torch.randn(16, 8).pin_memory() for _ in range(8)]
    ys = [torch.randint(0, 8, (16,)).pin_memory() for _ in range(8)]
    harness("micro_mlp", mlp, xs, ys, 100 if quick else 400, 3 if quick else 5)

    model = resnet18().to(device)
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local])
    xs = [torch.randn(64, 3, 224, 224).pin_memory() for _ in range(2)]
    ys = [torch.randint(0, 10, (64,)).pin_memory() for _ in range(2)]
    harness("resnet18_b64", model, xs, ys, 8 if quick else 24, 2 if quick else 3)

    # live render tick (StepCombined / step-memory twins) across the job's ranks, next to the
    # reference's computation (oracle port, rows pre-parsed: no SQLite / JSON) on rank 0
    try:
        import torch.distributed as dist
        from oracle import live_oracle
        from traceml_b200 import records as rec_mod
        import replay
        from traceml_b200.engine import Engine
        from traceml_b200.live import StepCombinedComputer, StepMemoryCombinedComputer
        from traceml_b200.reduce import LocalComm, TorchDistComm

        rank = dist.get_rank() if world > 1 else 0
        S = 2000
        mine = replay.make_step_replay("input_straggler", world, S, seed=3, only_ranks=[rank])[rank]
        le = Engine(device=local, rank=rank, world=world, ring_slots=4096, proc_slots=64)
        le.load_steps(mine)
        torch.cuda.synchronize(device)
        comm = TorchDistComm() if world > 1 else LocalComm()
        tick_t = StepCombinedComputer([le], comm, window_size=100)
        tick_m = StepMemoryCombinedComputer([le], comm, window_size=400)

        def tick_ms(fn, n=30):
            for _ in range(3):
                fn()
            ts = []
            for _ in range(n):
                t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
            return statistics.median(ts)

        live = {"step_time_cli_ms": tick_ms(tick_t.compute_cli),
                "step_time_dashboard_ms": tick_ms(tick_t.compute_dashboard),
                "step_memory_ms": tick_ms(tick_m.compute), "ranks": world,
                "window": {"step_time": 100, "step_memory": 400}}
        le.close()
        if rank == 0:
            allr = replay.make_step_replay("input_straggler", world, S, seed=3)
            rows = {r: [rec_mod.step_record_to_wire(x, device=f"cuda:{r}") for x in allr[r][-400:]]
                    for r in allr}
            mrows = {r: [(int(s_), float(a_), float(v_)) for s_, a_, v_ in
                         zip(allr[r]["step"], allr[r]["peak_alloc"], allr[r]["peak_resv"])] for r in allr}
            live["reference_port_step_time_cli_ms"] = tick_ms(
                lambda: live_oracle.live_step_time(rows, window=100), n=5)
            live["reference_port_step_memory_ms"] = tick_ms(
                lambda: live_oracle.live_step_memory(mrows, window=400), n=5)
        out["live_tick"] = live
    except Exception as exc:
        out["live_tick"] = {"error": f"{type(exc).__name__}: {exc}"}
    return out


# ----------------------------------------------------------------------------- reference arm
REF_LEGS = os.path.join(ROOT, "baseline", "reference_legs.py")
DEFAULT_W = 10_000          # the reference's default summary window (reporting/config.py:13)
DEFAULT_PROC_ROWS = 2_000


def ref_available() -> bool:
    return os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "traceml"))


def ref_leg(argv, timeout=1500) -> dict:
    """Run baseline/reference_legs.py (the UNMODIFIED reference from oracle/_ref) in its own
    process -- no module of this repository's engine is imported there -- and parse its JSON."""
    env = {k: v for k, v in os.environ.items()
           if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "GROUP_RANK", "MASTER_ADDR",
                        "MASTER_PORT", "TORCHELASTIC_RUN_ID", "PYTHONPATH")}
    try:
        p = subprocess.run([sys.executable, REF_LEGS] + [str(a) for a in argv], capture_output=True,
                           text=True, timeout=timeout, env=env, cwd=ROOT)
        lines = [ln for ln in p.stdout.strip().splitlines() if ln.startswith("{")]
        if p.returncode != 0 or not lines:
            return {"error": f"rc={p.returncode}: {(p.stderr or p.stdout)[-400:]}"}
        return json.loads(lines[-1])
    except Exception as exc:  # noqa: BLE001
        return {"error": f"{type(exc).__name__}: {exc}"}


def oracle_reduce_sample(R: int, W: int, seed: int = 1):
    """Fallback only (no oracle/_ref): the oracle port of the reference's CPU reduce."""
    import replay
    from helpers import oracle_mem_rows, oracle_proc_rows, oracle_time_rows
    from oracle import process_oracle, step_memory_oracle, step_time_oracle

    recs = replay.make_step_replay("balanced", R, W, seed)
    procs = replay.make_proc_replay("normal", R, 2000, seed)
    trows, mrows, prows = oracle_time_rows(recs, W), oracle_mem_rows(recs), oracle_proc_rows(procs, R)

    def once():
        t0 = time.perf_counter()
        step_time_oracle.step_time_section(trows, max_rows=W)
        step_memory_oracle.step_memory_section(mrows, window_size=W)
        process_oracle.process_section(prows, max_rows=W)
        return time.perf_counter() - t0

    return once


def workload_config(R: int, W: int) -> dict:
    """The `config` both arms report, key for key: the workload is the same; the reference arm
    times a bounded sample of it (described under ``cpu_baseline.sample``, not here)."""
    return {"workload": f"BASELINE config 4 reduce-stress replay: R={R} ranks x W={W} step "
                        "records/rank (128 B) + 60000 process samples/rank; full window "
                        "reduce + diagnosis per step",
            "window": W, "ranks": R,
            "l2": "inputs larger than L2 (ring 512 MB/rank at W=4e6); no flush needed",
            "algorithmic_bytes_per_step": b_reduce(R, W)}


def summary_digest(sections: dict) -> dict:
    """The comparable core of a summary, same shape from either arm: status per section and the
    public rollups ``global.{median,worst}`` = {metric: {value, idx}} (a15 / a16)."""
    out = {}
    for name in ("step_time", "step_memory", "process"):
        sec = sections.get(name) or {}
        g = sec.get("global") or {}
        out[name] = {"status": sec.get("status"),
                     "median": {k: v for k, v in (g.get("median") or {}).items()},
                     "worst": {k: v for k, v in (g.get("worst") or {}).items()}}
    return out


def compare_digests(mine: dict, ref: dict, rel: float = 1e-9) -> dict:
    """status and idx exact, values within ``rel`` (SURVEY 8d tolerances)."""
    bad, checked = [], 0
    for name in ("step_time", "step_memory", "process"):
        a, b = mine.get(name) or {}, ref.get(name) or {}
        if a.get("status") != b.get("status"):
            bad.append(f"{name}.status {a.get('status')!r} != {b.get('status')!r}")
        checked += 1
        for roll in ("median", "worst"):
            for metric, rv in (b.get(roll) or {}).items():
                mv = (a.get(roll) or {}).get(metric)
                if mv is None:
                    if name != "process":  # process rollups are compared where both sides emit them
                        bad.append(f"{name}.{roll}.{metric} missing")
                    continue
                checked += 1
                if str(mv.get("idx")) != str(rv.get("idx")):
                    bad.append(f"{name}.{roll}.{metric}.idx {mv.get('idx')} != {rv.get('idx')}")
                x, y = mv.get("value"), rv.get("value")
                if (x is None) != (y is None) or (x is not None and abs(float(x) - float(y)) > rel * max(abs(float(y)), 1e-300)):
                    bad.append(f"{name}.{roll}.{metric}.value {x!r} !~ {y!r}")
    return {"ok": not bad, "fields_checked": checked, "mismatches": bad[:8]}


def run_reference(args, rank, world):
    if rank != 0:
        return
    R = max(1, args.gpus)
    W = int(args.window)
    K, Wm = max(1, args.steps), max(0, args.warmup)
    # Bounded sample per step, sized by K so that the whole run ends within minutes whatever
    # --steps says: the reference costs ~100 us per row (single-threaded Python), so K + W steps of
    # `rows` rows take (K + W) * rows * 1e-4 s; aim at ~100 s in all, never above --sample rows.
    budget_rows = int(100.0 / 1.0e-4 / (K + Wm))
    Ws = max(500, min(args.sample, budget_rows) // R)
    line = {
        "impl": "reference", "metric": "cross_rank_reduce_GBps", "unit": "GB/s", "n_gpus": args.gpus,
        "steps": K, "warmup": Wm, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f64", "data": "synthetic", "config": workload_config(R, W), "host_cores": os.cpu_count(),
    }
    if ref_available():
        red = ref_leg(["--leg", "reduce", "--ranks", R, "--rows", Ws, "--steps", K, "--warmup", Wm,
                       "--proc-rows", DEFAULT_PROC_ROWS])
        if "error" in red:
            print(json.dumps({"impl": "reference", "unavailable": red["error"][:300]}))
            return
        t = sum(red["s_per_step"]) / len(red["s_per_step"])
        val = b_reduce(R, Ws) / t / 1e9
        line.update({
            "value": val, "ms_per_step": t * 1e3,
            "cpu_baseline": {
                "value": val, "unit": "GB/s", "cores": 1, "kind": "reference",
                "sample": f"each step = the UNMODIFIED reference (oracle/_ref, own process): "
                          f"StepTime/StepMemory/Process SummarySection.build(db) on R={R} ranks x {Ws} rows of the "
                          f"workload, SQLite written by the reference's own projection writers; "
                          f"{red['us_per_row']:.1f} us/row, single-threaded Python (1 of {os.cpu_count()} cores)",
                "sections_s": red["s_sections_median"], "sqlite_projection": red["sqlite_projection"]},
            "e2e": {"value": val, "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "reference_version": red.get("reference_version"),
        })
        # the reference's own default window, full size, same seed as the product arm's leg
        dw = ref_leg(["--leg", "reduce", "--ranks", R, "--rows", DEFAULT_W, "--window", DEFAULT_W,
                      "--steps", 1, "--warmup", 0, "--proc-rows", DEFAULT_PROC_ROWS])
        if "error" not in dw:
            line["default_window"] = {
                "window": DEFAULT_W, "ranks": R, "ms": dw["s_per_step_median"] * 1e3,
                "GBps": b_reduce(R, DEFAULT_W) / dw["s_per_step_median"] / 1e9,
                "summary": summary_digest(dw["summary"]), "same_config_as_product_arm": True}
        else:
            line["default_window"] = dw
        if torch.cuda.is_available() and not args.no_overhead:
            line["step_overhead"] = ref_leg(["--leg", "overhead", "--quick"])
    else:
        once = oracle_reduce_sample(R, Ws)
        for _ in range(Wm):
            once()
        times = [once() for _ in range(K)]
        t = sum(times) / len(times)
        val = b_reduce(R, Ws) / t / 1e9
        line.update({
            "value": val, "ms_per_step": t * 1e3,
            "cpu_baseline": {"value": val, "unit": "GB/s", "cores": 1, "kind": "port",
                             "sample": f"oracle/_ref missing: oracle port, R={R} x W={Ws} rows pre-parsed"},
            "e2e": {"value": val, "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}})
    print(json.dumps(line))


# ----------------------------------------------------------------------------- parity (outside timing)
def _gather(obj, world):
    if world <= 1:
        return [obj]
    out = [None] * world
    torch.distributed.all_gather_object(out, obj)
    return out


def parity_check(recs, res, W, rank, world, device, ram_total):
    """The W-sized result of THIS run against the numpy oracle on the same seed.

    Every rank restates its own window with numpy (reference-order sums, exact integer memory
    sums); rank 0 assembles the sections through the pinned row-level oracle's own rule code.
    Series: every step at N = 1; at N > 1 a strided sample plus the last 10 000 steps (all the
    trend rules read) of every rank's shard -- the rows are gathered, not regenerated."""
    from helpers import assert_struct, plain, strip_device
    from oracle import fast_oracle as fo

    t0 = time.perf_counter()
    part = fo.rank_part(recs, W)
    mem = fo.mem_part(recs, W)
    red = res["reduce"]
    n = int(red.time.n_common)
    steps = part["steps"] if part else np.zeros(0, np.int64)
    bounds = _gather((int(steps[0]) if steps.size else None, int(steps[-1]) if steps.size else None,
                      int(steps.size)), world)
    lock_step = all(b == bounds[0] for b in bounds) and bounds[0][2] > 0 and \
        bounds[0][1] - bounds[0][0] + 1 == bounds[0][2] and n == bounds[0][2]
    if not lock_step:
        return {"checked": False, "why": "ranks not in lock step: the numpy oracle's gathered-sample mode covers "
                                         "the bench replay only"}
    common = steps
    al = fo.aligned_part(part, common)
    # sampled steps: everything at N = 1, else stride + tail
    if world == 1:
        idx = np.arange(n)
    else:
        stride = max(1, n // 200_000)
        idx = np.unique(np.concatenate([np.arange(0, n, stride), np.arange(max(0, n - fo.TAIL), n)]))
    ser = red.time.series  # [16, n] device view, this rank's shard valid
    lo, hi = red.time.shard if getattr(red.time, "shard", None) else (0, n)
    mine = idx[(idx >= lo) & (idx < hi)]
    dev_vals = ser[:, torch.from_numpy(mine).to(device)].cpu().numpy() if mine.size else np.zeros((16, 0))
    payload = {
        "summary": part["summary"], "n": part["n"], "aligned": al["summary"],
        "rows": al["rows"][idx], "series_idx": mine, "series_vals": dev_vals,
        "mem_sum": (int(mem["alloc"].sum(dtype=np.uint64)), int(mem["resv"].sum(dtype=np.uint64))) if mem else None,
        "mem_peak": (int(mem["alloc"].max()), int(mem["resv"].max())) if mem else None,
        "latest": int(recs["step"].max()),
    }
    allp = _gather(payload, world)
    if rank != 0:
        return None
    R = world
    ser_ref = fo.series16(np.stack([p["rows"] for p in allp]))          # [16, len(idx)]
    got = np.full((16, idx.size), np.nan)
    pos = {int(v): k for k, v in enumerate(idx.tolist())}
    for p in allp:
        cols = [pos[int(v)] for v in p["series_idx"].tolist()]
        got[:, cols] = p["series_vals"]
    series_equal = bool(np.array_equal(got, ser_ref))
    n_bad = int((got != ser_ref).sum())
    tail = min(fo.TAIL, n)
    tail_cols = [pos[v] for v in range(n - tail, n)]
    parts = {r: {"summary": allp[r]["summary"]} for r in range(R)}
    aligned = {r: {"summary": allp[r]["aligned"]} for r in range(R)}
    ref_t = fo.step_time_from_parts(parts, aligned, n, int(common[0]), int(common[-1]), W,
                                    ser_ref[:, tail_cols], common[n - tail:], max(p["latest"] for p in allp))
    bad = []

    def chk(a, b, what, rel=1e-9):
        try:
            assert_struct(plain(a), plain(b), what, rel)
        except AssertionError as exc:
            bad.append(str(exc)[:200])

    gt = res["step_time"]
    chk(gt["data"]["aligned_window"], ref_t["data"]["aligned_window"], "time.window")
    chk(gt["data"]["aligned_summary"], ref_t["data"]["aligned_summary"], "time.aligned_summary")
    chk(gt["data"]["per_global_rank_summary"], ref_t["data"]["per_global_rank_summary"], "time.per_rank_summary")
    chk(gt["diagnosis"], ref_t["diagnosis"], "time.diagnosis")
    chk(gt["global"], ref_t["global"], "time.global")
    chk(gt["overview"], ref_t["overview"], "time.overview")
    sums_bit_exact = all(plain(gt["data"]["aligned_summary"]).get(str(r)) == plain(ref_t["data"]["aligned_summary"]).get(str(r))
                         for r in range(R))
    # step memory: means from exact integer sums, peaks, series columns 12..15
    from oracle import step_memory_oracle as smo

    gm = res["step_memory"]
    means = {str(r): {"peak_allocated_bytes": float(allp[r]["mem_sum"][0]) / n,
                      "peak_reserved_bytes": float(allp[r]["mem_sum"][1]) / n} for r in range(R)
             if allp[r]["mem_sum"] is not None}
    chk(gm["per_global_rank"], means, "mem.per_rank_means")
    chk(gm["global"], smo.rollup_points(means), "mem.global")
    metrics = []
    for i, name in enumerate(("peak_allocated", "peak_reserved")):
        peaks = [float(allp[r]["mem_peak"][i]) for r in range(R)]
        med_peak, worst_peak = float(smo.median2(peaks)), float(max(peaks))
        metrics.append({"metric": name,
                        "series": {"steps": [int(s) for s in common[n - tail:]],
                                   "median": ser_ref[12 + 2 * i, tail_cols].tolist(),
                                   "worst": ser_ref[13 + 2 * i, tail_cols].tolist()},
                        "summary": {"window_size": W, "steps_used": n, "median_peak": med_peak, "worst_peak": worst_peak,
                                    "worst_rank": int(peaks.index(worst_peak)),
                                    "skew_ratio": float(worst_peak / med_peak if med_peak > 0 else 0.0),
                                    "skew_pct": float((worst_peak - med_peak) / med_peak if med_peak > 0 else 0.0)},
                        "coverage": {"expected_steps": W, "steps_used": n, "completed_step": int(common[-1]),
                                     "world_size": R, "ranks_present": R, "incomplete": False}})
    ref_md = strip_device(smo.diagnose_summary(metrics, gm.get("gpu_total_bytes")))
    gd = strip_device(plain(gm["diagnosis"]))
    chk(gd["primary"], ref_md["primary"], "mem.diagnosis.primary")
    chk(gd["issues"], ref_md["issues"], "mem.diagnosis.issues")
    return {
        "checked": True, "ok": (not bad) and series_equal, "window": W, "ranks": R,
        "oracle": "oracle/fast_oracle.py (numpy; pinned == row-level oracle == unmodified reference)",
        "labels": {"step_time": (ref_t["diagnosis"] or {}).get("primary", {}).get("status"),
                   "step_memory": ref_md["primary"]["status"]},
        "idx": {"median_total_step": ref_t["global"]["median"]["total_step_ms"]["idx"],
                "worst_total_step": ref_t["global"]["worst"]["total_step_ms"]["idx"]},
        "aligned_window": {k: ref_t["data"]["aligned_window"][k] for k in ("steps_analyzed", "start_step", "end_step")},
        "series": {"steps_checked": int(idx.size), "of": n, "mode": "all" if world == 1 else "stride+tail",
                   "bit_equal": series_equal, "elements_differing": n_bad},
        "per_rank_sums_bit_exact": bool(sums_bit_exact),
        "mismatches": bad[:8], "seconds": time.perf_counter() - t0,
    }


def default_window_leg(rank, local, world, device, comm):
    """The reference's default window (W = 10^4) on the seed the reference arm uses: this engine's
    time per reduce and -- on rank 0, in a separate process -- the UNMODIFIED reference's, with the
    two summaries compared field by field."""
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    recs = replay.make_step_replay("balanced", world, DEFAULT_W, seed=1, only_ranks=[rank])[rank]
    procs = replay.make_proc_replay("normal", world, DEFAULT_PROC_ROWS, seed=1, only_ranks=[rank])[rank]
    eng = Engine(device=local, rank=rank, world=world, ring_slots=int(DEFAULT_W * 1.5), proc_slots=4096)
    eng.load_steps(recs); eng.load_procs(procs)
    torch.cuda.synchronize(device)
    summ = sections.SummaryEngine([eng], comm, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=world)
    for _ in range(5):
        res = summ.build(DEFAULT_W, DEFAULT_W)
    barrier(world); torch.cuda.synchronize(device)
    n_it = 50
    t0 = time.perf_counter()
    for _ in range(n_it):
        res = summ.build(DEFAULT_W, DEFAULT_W)
    torch.cuda.synchronize(device)
    ms = max_over_ranks((time.perf_counter() - t0) / n_it * 1e3, world, device)
    out = None
    if rank == 0:
        mine = {"step_time": {"status": res["step_time"]["diagnosis"]["primary"]["status"], "global": res["step_time"]["global"]},
                "step_memory": {"status": res["step_memory"]["diagnosis"]["primary"]["status"],
                                "global": res["step_memory"]["global"]},
                "process": {"status": res["process"]["primary"]["status"], "global": res["process"].get("global")}}
        out = {"window": DEFAULT_W, "ranks": world, "ms": ms, "GBps": b_reduce(world, DEFAULT_W) / (ms * 1e-3) / 1e9,
               "summary": summary_digest(mine), "same_config_as_reference_arm": True}
        if ref_available():
            dw = ref_leg(["--leg", "reduce", "--ranks", world, "--rows", DEFAULT_W, "--window", DEFAULT_W,
                          "--steps", 1, "--warmup", 0, "--proc-rows", DEFAULT_PROC_ROWS])
            if "error" in dw:
                out["reference"] = dw
            else:
                out["reference"] = {"ms": dw["s_per_step_median"] * 1e3, "us_per_row": dw["us_per_row"],
                                    "kind": "unmodified reference, oracle/_ref, separate process, 1 core"}
                out["speedup_vs_reference"] = dw["s_per_step_median"] * 1e3 / ms
                out["parity_vs_reference"] = compare_digests(out["summary"], summary_digest(dw["summary"]))
    barrier(world)
    eng.close()
    return out


# ----------------------------------------------------------------------------- --dump-outputs
DUMP_SERIES_COLS = 1 << 17  # sampled steps per series over all ranks: 16 x 2^17 float64 = 16 MB


def _flatten_numbers(obj, vals):
    """Every numeric leaf of a section dict, in sorted-key order (strings are labels and None marks
    a value the section does not have: both skipped)."""
    if isinstance(obj, dict):
        for k in sorted(obj, key=str):
            _flatten_numbers(obj[k], vals)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _flatten_numbers(v, vals)
    elif isinstance(obj, (bool, int, float, np.integer, np.floating)):
        vals.append(float(obj))


def capture_outputs(res, world: int, seed: int = 0) -> dict:
    """What one ``SummaryEngine.build`` handed its caller, as float64 host arrays: the numbers of
    the three sections and the per-step median / worst series (a fixed, seeded sample of the
    steps when the window is larger than DUMP_SERIES_COLS, with the sampled step indices).  Each of
    the ``world`` ranks samples its own shard, DUMP_SERIES_COLS / world steps of it, so that the
    files of all ranks together stay within the same size."""
    out = {}
    for name in ("step_time", "step_memory", "process"):
        vals = []
        _flatten_numbers(res.get(name), vals)
        out[name] = np.asarray(vals, dtype=np.float64)
    seen = set()
    for kind in ("time", "mem"):
        k = getattr(res["reduce"], kind)
        if k.series is None or not k.n_common or k.series.data_ptr() in seen:
            continue
        seen.add(k.series.data_ptr())
        lo, hi = k.shard if k.shard[1] > k.shard[0] else (0, int(k.n_common))
        take = min(hi - lo, max(1, DUMP_SERIES_COLS // world))
        cols = lo + np.sort(np.random.default_rng(seed).choice(hi - lo, take, replace=False))
        idx = torch.from_numpy(cols).to(k.series.device)
        out[f"{kind}_series"] = k.series[:, idx].double().cpu().numpy()
        out[f"{kind}_series_steps"] = cols.astype(np.float64)
    return out


def write_outputs(outdir: str, arrays: dict, rank: int, world: int) -> None:
    os.makedirs(outdir, exist_ok=True)
    for name, arr in arrays.items():
        np.save(os.path.join(outdir, f"{name}.npy" if world == 1 else f"{name}_rank{rank}.npy"), arr)


# ----------------------------------------------------------------------------- main arm
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--window", type=int, default=4_000_000, help="W: step records per rank")
    ap.add_argument("--sample", type=int, default=40_000, help="cpu-baseline rows per rank")
    ap.add_argument("--exchange", default="auto", choices=["auto", "p2p", "nccl", "a2a"])
    ap.add_argument("--no-overhead", action="store_true")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (float64)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    args.warmup = max(3, args.warmup) if args.impl == "b200" else args.warmup

    if args.impl == "reference":
        rank = int(os.environ.get("RANK", "0"))
        run_reference(args, rank, int(os.environ.get("WORLD_SIZE", "1")))
        return

    rank, local, world = dist_setup()
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine
    from traceml_b200.reduce import LocalComm, TorchDistComm

    t_bench0 = time.perf_counter()
    W = int(args.window)
    R = world
    comm = TorchDistComm() if world > 1 else LocalComm()

    # ---- synthetic inputs of BASELINE config 4's shape, one rank's worth, in pinned host memory
    recs = replay.make_step_replay("balanced", R, W, seed=1, only_ranks=[rank])[rank]
    procs = replay.make_proc_replay("normal", R, 60_000, seed=1, only_ranks=[rank])[rank]
    host = torch.empty(W * 128, dtype=torch.uint8).pin_memory()
    host.numpy()[:] = recs.view(np.uint8).reshape(-1)
    eng = Engine(device=local, rank=rank, world=R, ring_slots=W, proc_slots=65_536)
    eng.load_procs(procs)
    stream = torch.cuda.current_stream(device)
    eng.load_steps_ptr(host.data_ptr(), W, stream.cuda_stream)
    torch.cuda.synchronize(device)
    summ = sections.SummaryEngine([eng], comm, exchange=args.exchange,
                                  ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R)

    # ---- (1) device-resident reduce: K steps, CUDA events, max over ranks
    # (clock sampling starts before the warm-up steps -- same workload -- because the
    # timed region itself is only a few ms long, shorter than one nvidia-smi period)
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    for _ in range(args.warmup):
        res = summ.build(W, 60_000)
    barrier(world); torch.cuda.synchronize(device)
    l0 = eng.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stage = {}
    e0.record()
    for _ in range(args.steps):
        res = summ.build(W, 60_000)
        for k, v in res["reduce"].timings_ms.items():
            stage.setdefault(k, []).append(v)
    e1.record()
    torch.cuda.synchronize(device); barrier(world)
    launches = eng.launch_count - l0
    # the series are views of the engine's workspace: copy them out before the next build
    dumped = capture_outputs(res, world) if args.dump_outputs else None
    # stage breakdown (a diagnostic, outside the timed region: it adds a dozen torch events
    # per step).  The two kernels' own times (k3a, k4) above come from the timed steps.
    for _ in range(max(3, args.steps // 2)):
        r2 = summ.build(W, 60_000, timings=True)
        for k, v in r2["reduce"].timings_ms.items():
            if k not in ("k3a", "k4"):
                stage.setdefault(k, []).append(v)
    torch.cuda.synchronize(device); barrier(world)
    clk = None
    if rank == 0:
        t_wait = time.time()
        while not clocks.lines and time.time() - t_wait < 1.5:   # at least one sample under load
            summ.build(W, 60_000)
        clk = clocks.stop()
    ms_total = max_over_ranks(e0.elapsed_time(e1), world, device)
    ms_step = ms_total / args.steps
    value = b_reduce(R, W) / (ms_step * 1e-3) / 1e9
    # a longer look at the same loop (>= 1 s), as a cross-check of the K-step figure
    barrier(world); torch.cuda.synchronize(device)
    n_sus = max(50, int(1000.0 / max(ms_step, 1e-3)))
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(n_sus):
        res = summ.build(W, 60_000)
    s1.record()
    torch.cuda.synchronize(device)
    sustained = {"steps": n_sus, "ms_per_step": max_over_ranks(s0.elapsed_time(s1), world, device) / n_sus}
    barrier(world)

    # ---- parity of THIS window against the numpy oracle (outside the timed region)
    parity = None
    if not args.no_parity:
        try:
            parity = parity_check(recs, res, W, rank, world, device, replay.PROC_RAM_TOTAL_BYTES)
        except Exception as exc:  # noqa: BLE001 -- a failed check is reported, never hidden
            parity = {"checked": False, "error": f"{type(exc).__name__}: {exc}"[:300]}
        barrier(world)
    del recs

    # ---- roofline of the dominant kernels (per launch, this rank)
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    peak, peak_src = 3350.0, "H100 SXM data sheet: 3.35 TB/s HBM3"
    if os.path.exists(peaks_path):
        with open(peaks_path) as fh:
            peak = float(json.load(fh)["hbm_gbs"]); peak_src = "measured (MEASURED_PEAKS.json hbm_gbs, burst)"
    med = {k: statistics.median(v) for k, v in stage.items()}
    n_shard = W // R
    k4_bytes = R * n_shard * 64.0 + 128.0 * n_shard          # rows read + 16 series written
    k3a_bytes = W * (128.0 + 64.0 + 8.0 + 1.0)               # record read, row + step id + flags written
    kernels = {
        "k_window_reduce": {"ms": med.get("k4"), "bytes": k4_bytes,
                            "GBps": k4_bytes / (med["k4"] * 1e-3) / 1e9 if med.get("k4") else None},
        "k_window_rows": {"ms": med.get("k3a"), "bytes": k3a_bytes,
                          "GBps": k3a_bytes / (med["k3a"] * 1e-3) / 1e9 if med.get("k3a") else None},
    }
    if getattr(res["reduce"], "fused_rows", False):
        # single rank: ring -> series in one kernel; 128 B record read + 16 series x 8 B written per step
        fb = W * 256.0
        kernels = {"k_window_fused": {"ms": med.get("k3a"), "bytes": fb,
                                      "GBps": fb / (med["k3a"] * 1e-3) / 1e9 if med.get("k3a") else None}}
    if R > 1 and med.get("k4"):
        # step-sharded K4 loads (R-1)/R of its rows from peer HBM: NVLink 4 is its bound, not the
        # local HBM.  Denominator: the H100 SXM data sheet's 900 GB/s per GPU, 450 per direction
        nv = (R - 1) * n_shard * 64.0
        kernels["k_window_reduce"]["nvlink"] = {
            "bytes_in": nv, "GBps": nv / (med["k4"] * 1e-3) / 1e9, "peak": 450.0, "nominal": 900.0,
            "frac": nv / (med["k4"] * 1e-3) / 1e9 / 450.0,
            "peak_source": "H100 SXM data sheet, NVLink 4, one direction"}
    dom = max(kernels, key=lambda k: kernels[k]["ms"] or 0.0)
    roofline = {"bound": "hbm", "kernel": dom, "achieved": kernels[dom]["GBps"], "peak": peak,
                "unit": "GB/s", "frac": (kernels[dom]["GBps"] or 0.0) / peak, "traffic": None,
                "peak_source": peak_src, "kernels": kernels, "stage_ms": med}

    # ---- (2) end to end from HOST buffers: H2D + reduce + results on the host
    def e2e_once():
        eng.reset()
        eng.load_procs(procs)
        eng.load_steps_ptr(host.data_ptr(), W, stream.cuda_stream)
        return summ.build(W, 60_000)

    for _ in range(2):
        e2e_once()
    barrier(world); torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        res = e2e_once()
    torch.cuda.synchronize(device)
    e2e_s = max_over_ranks(time.perf_counter() - t0, world, device) / args.steps
    barrier(world)
    e2e = {"value": b_reduce(R, W) / e2e_s / 1e9, "unit": "GB/s",
           "h2d_bytes_per_step": (W * 128 + 60_000 * 64) * R,
           # per rank: prepare results 616 B + process aggregates 128 B + band sums 1024 B, and at
           # R > 1 the gathered exchange vectors (64 + 128 doubles per rank, read back on every rank)
           "d2h_bytes_per_step": (1_768 + (1_536 * R if R > 1 else 0)) * R,
           "ms_per_step": e2e_s * 1e3}

    exchange_used = res["reduce"].exchange
    diagnosis = res["step_time"]["diagnosis"]["primary"]["status"] if res["step_time"]["diagnosis"] else None
    eng.close()

    # ---- (3) the reference's default window, both arms, same seed
    try:
        default_window = default_window_leg(rank, local, world, device, comm)
    except Exception as exc:  # noqa: BLE001
        default_window = {"error": f"{type(exc).__name__}: {exc}"[:300]}

    # ---- (4) per-step overhead leg (the reference's real trace_step: own process, rank 0, N = 1)
    overhead = None
    if not args.no_overhead:
        overhead = step_overhead(device, world, local)
        if rank == 0 and world == 1 and ref_available():
            from traceml_b200.runtime import shutdown_engine

            shutdown_engine()
            ro = ref_leg(["--leg", "overhead"])
            overhead["reference"] = ro
            for k in ("micro_mlp", "resnet18_b64"):
                if k in ro and k in overhead:
                    overhead[k]["reference_us"] = ro[k]["reference_us"]
                    overhead[k]["reference_untraced_us"] = ro[k]["untraced_us"]
                    overhead[k]["reference_overhead_us"] = ro[k]["reference_overhead_us"]

    # ---- (5) CPU baseline on a bounded sample (rank 0, N = 1 only): the unmodified reference
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        if ref_available():
            red = ref_leg(["--leg", "reduce", "--ranks", 1, "--rows", args.sample, "--steps", 3, "--warmup", 1,
                           "--proc-rows", DEFAULT_PROC_ROWS])
            if "error" not in red:
                t = red["s_per_step_median"]
                cpu = {"value": b_reduce(1, args.sample) / t / 1e9, "unit": "GB/s", "cores": 1, "kind": "reference",
                       "sample": f"R=1 x W={args.sample} rows of the same workload ({t:.2f} s/step, "
                                 f"{red['us_per_row']:.1f} us/row): the UNMODIFIED reference's three summary sections "
                                 "over SQLite written by its own projection writers (oracle/_ref, own process)",
                       "host_cores": os.cpu_count(), "sqlite_projection": red["sqlite_projection"]}
            else:
                cpu = {"error": red["error"], "kind": "reference"}
        if cpu is None or "error" in cpu:
            once = oracle_reduce_sample(1, args.sample)
            once()
            t = once()
            cpu = {"value": b_reduce(1, args.sample) / t / 1e9, "unit": "GB/s", "cores": 1, "kind": "port",
                   "sample": f"R=1 x W={args.sample} rows ({t:.2f} s, {t / args.sample * 1e6:.1f} us/row); "
                             "oracle port of the reference's Python reduce, rows pre-parsed (no SQLite/JSON)",
                   "host_cores": os.cpu_count()}

    if rank == 0:
        line = {
            "metric": "cross_rank_reduce_GBps", "value": value, "unit": "GB/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "synthetic",
            "config": workload_config(R, W), "exchange": exchange_used,
            "clocks": clk, "e2e": e2e, "gpu_launches": int(launches),
            "records_per_s": R * W / (ms_step * 1e-3), "sustained": sustained,
            "parity": parity, "default_window": default_window,
            "scaling_note": "weak: every rank holds W records; by the SURVEY formula the bytes grow as "
                            "(64 R + 128) W, so constant step time gives value(N)/value(1) = (64 N + 128)/192",
            "roofline": roofline, "cpu_baseline": cpu, "step_overhead": overhead,
            "diagnosis": diagnosis, "bench_wall_s": time.perf_counter() - t_bench0,
        }
        print(json.dumps(line))
    if dumped is not None:
        write_outputs(args.dump_outputs, dumped, rank, world)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
