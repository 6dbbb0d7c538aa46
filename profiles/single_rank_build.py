"""Where the time of one single-rank summary build goes, next to what the HBM can do.

Builds the workload ``bench.py --gpus 1`` times (same replay kinds and seed, ``Engine(ring_slots=W)``,
steps loaded from pinned memory with ``load_steps_ptr``, 60 000 process samples) and prints one JSON
line:

  * ``build_ms``: CUDA events around K back-to-back ``SummaryEngine.build`` calls, per call;
  * ``build_wall_ms``: host clock around one call (it ends in a stream synchronise), median;
  * ``stage_ms``: the native driver's own stage times and ``k3a`` (the fused pass), medians;
  * ``sections_json_ms``: the host time of ``tml_sections_json`` alone, and ``python_rest_ms``,
    what is left of the wall time after the native driver and the JSON emitter;
  * ``segments_ms``: host time of each segment of a build (medians): Python entry -> native call,
    native call -> pass submitted, -> return from the wait, native collect, sections JSON, the
    Python after it;
  * ``kernel_ms``: device time per build of each kernel (torch.profiler, a run of its own), and
    ``device_idle_ms``: ``build_ms`` minus the pass and the band kernel;
  * ``timeline_ms``: the device timeline around one build (torch.profiler, another run of its own):
    pass end -> ``k_bands`` start, ``k_bands`` end -> last copy end, last copy end -> next pass start;
  * ``copy_ceiling``: ``dst.copy_(src)`` on 512 MB device tensors (1.024 GB moved), CUDA events,
    median of 25 after warm-up; the fused pass against it, counting the bytes it moves by the stream
    that ran (``stream``): 32 B per step for a packed-streamable window (the ring's packed records),
    64 B for another certified one (the hot halves), 65 B otherwise (the hot halves and the memory
    bytes), plus W * 64 of series when each median / worst series pair is stored once
    (``series_paired``), W * 128 otherwise;
  * ``gpu``: card name, power limit and max SM clock (read-only ``nvidia-smi`` query).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROC_ROWS = 60_000


def gpu_info(index: int = 0) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clk}
    except Exception as exc:  # noqa: BLE001 -- reported, not hidden
        return {"error": f"{type(exc).__name__}: {exc}"[:200]}


def copy_ceiling(torch, nbytes: int = 512_000_000, reps: int = 25) -> dict:
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda").random_(0, 255)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        dst.copy_(src)
        b.record()
    torch.cuda.synchronize()
    ms = statistics.median(a.elapsed_time(b) for a, b in ev)
    del src, dst
    torch.cuda.empty_cache()
    return {"bytes_moved": 2 * nbytes, "ms": ms, "GBps": 2 * nbytes / (ms * 1e-3) / 1e9}


def segments(summ, W: int, steps: int) -> dict:
    """Host time of each segment of one build, medians over ``steps`` builds.  The native entry points
    are wrapped to stamp their calls; the driver's own stage times split the reduce inside them:
    ``reduce`` is its host time up to the submission of the pass (0 where a driver does not report
    it), ``prepare`` up to the return from the wait, ``bands`` the collect after it."""
    from traceml_b200 import _abi

    lib = _abi.lib()
    stamps: list = []
    wrapped = {}
    for name in ("tml_summary_run_", "tml_reduce_run", "tml_sections_json"):
        fn = getattr(lib, name, None)
        if fn is None:
            continue

        def stamp(*a, _fn=fn):
            t0 = time.perf_counter()
            rc = _fn(*a)
            stamps.append((t0, time.perf_counter()))
            return rc

        wrapped[name] = fn
        setattr(lib, name, stamp)
    keys = ("python_to_native", "native_launch", "launch_to_wait_return", "native_collect", "sections_json",
            "python_rest", "wall")
    rows: dict = {k: [] for k in keys}
    try:
        for _ in range(steps):
            stamps.clear()
            t0 = time.perf_counter()
            res = summ.build(W, PROC_ROWS)
            t1 = time.perf_counter()
            st = res["reduce"].timings_ms
            before = (stamps[0][0] - t0) * 1e3
            native = sum(b - a for a, b in stamps) * 1e3
            rows["python_to_native"].append(before)
            rows["native_launch"].append(st["reduce"])
            rows["launch_to_wait_return"].append(st["prepare"] - st["reduce"])
            rows["native_collect"].append(st["bands"])
            rows["sections_json"].append(native - st["total"])
            rows["python_rest"].append((t1 - t0) * 1e3 - before - native)
            rows["wall"].append((t1 - t0) * 1e3)
    finally:
        for name, fn in wrapped.items():
            setattr(lib, name, fn)
    return {k: statistics.median(v) for k, v in rows.items()}


def kernel_times(torch, summ, W: int, n: int = 30) -> dict:
    """Device time per build of each of the library's kernels (``k_*``), from torch.profiler over
    ``n`` builds: a run of its own, since tracing slows the host."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            summ.build(W, PROC_ROWS)
        torch.cuda.synchronize()
    out: dict = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0]
        if name.startswith("k_"):
            out[name] = out.get(name, 0.0) + e.device_time_total / 1e3 / n
    return out


def timeline_gaps(torch, summ, W: int, n: int = 30, trace_path: str = "") -> dict:
    """The device timeline around one build, from a torch.profiler trace of ``n`` back-to-back builds
    (a run of its own).  Per build, medians in ms:

      * ``pass_end_to_bands``: the fused pass's end -> ``k_bands``' start;
      * ``bands_to_last_copy``: ``k_bands``' end -> the end of the last device-to-host copy of the
        build (0 when no copy ends after ``k_bands``);
      * ``results_to_next_pass``: the later of those two ends -> the next build's pass start: the
        host round trip the GPU waits on.
    ``trace_path``: also write the Chrome trace there."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            summ.build(W, PROC_ROWS)
        torch.cuda.synchronize()
    if trace_path:
        prof.export_chrome_trace(trace_path)
    passes, bands, copies = [], [], []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        a, b = e.time_range.start / 1e3, e.time_range.end / 1e3  # us -> ms
        if "k_window_fused" in e.name:
            passes.append((a, b))
        elif "k_bands" in e.name:
            bands.append((a, b))
        elif "DtoH" in e.name or "Device -> Pinned" in e.name:
            copies.append((a, b))
    passes.sort(); bands.sort(); copies.sort()
    rows = {"pass_end_to_bands": [], "bands_to_last_copy": [], "results_to_next_pass": []}
    for (p0, p1), (q0, _) in zip(passes, passes[1:]):
        bd = [x for x in bands if p1 <= x[0] < q0]
        if not bd:
            continue
        b0, b1 = bd[0]
        ends = [c1 for c0, c1 in copies if p0 <= c0 < q0 and c1 > b1]
        last = max(ends) if ends else b1
        rows["pass_end_to_bands"].append(b0 - p1)
        rows["bands_to_last_copy"].append(last - b1)
        rows["results_to_next_pass"].append(q0 - last)
    out = {k: (statistics.median(v) if v else None) for k, v in rows.items()}
    out["builds"] = len(rows["results_to_next_pass"])
    out["copies_per_build"] = len(copies) / max(1, len(passes))
    return out


def measure(steps: int, window: int, warmup: int, trace: str = "") -> dict:
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch

    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine
    from traceml_b200.reduce import LocalComm

    assert torch.cuda.is_available(), "single_rank_build.py needs a CUDA device"
    torch.cuda.set_device(0)
    W = int(window)
    recs = replay.make_step_replay("balanced", 1, W, seed=1, only_ranks=[0])[0]
    procs = replay.make_proc_replay("normal", 1, PROC_ROWS, seed=1, only_ranks=[0])[0]
    host = torch.empty(W * 128, dtype=torch.uint8).pin_memory()
    host.numpy()[:] = recs.view(np.uint8).reshape(-1)
    eng = Engine(device=0, rank=0, world=1, ring_slots=W, proc_slots=65_536)
    eng.load_procs(procs)
    stream = torch.cuda.current_stream()
    eng.load_steps_ptr(host.data_ptr(), W, stream.cuda_stream)
    torch.cuda.synchronize()
    summ = sections.SummaryEngine([eng], LocalComm(), ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1)

    for _ in range(warmup):
        res = summ.build(W, PROC_ROWS)
    torch.cuda.synchronize()
    # (1) back-to-back builds between two events, as bench.py times them
    l0 = eng.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stage: dict = {}
    e0.record()
    for _ in range(steps):
        res = summ.build(W, PROC_ROWS)
        for k, v in res["reduce"].timings_ms.items():
            stage.setdefault(k, []).append(v)
    e1.record()
    torch.cuda.synchronize()
    build_ms = e0.elapsed_time(e1) / steps
    launches = (eng.launch_count - l0) / steps
    fused = bool(getattr(res["reduce"], "fused_rows", False))
    paired = bool(getattr(res["reduce"], "series_paired", False))
    # (2) host clock around single builds, and the JSON emitter alone on a fresh result
    wall = []
    for _ in range(steps):
        t0 = time.perf_counter()
        summ.build(W, PROC_ROWS)
        wall.append((time.perf_counter() - t0) * 1e3)
    o = summ.reducer.run_native(W, PROC_ROWS)
    sj = []
    for _ in range(steps):
        t0 = time.perf_counter()
        eng.sections_json(o, replay.PROC_RAM_TOTAL_BYTES, 1, W, PROC_ROWS)
        sj.append((time.perf_counter() - t0) * 1e3)
    seg = segments(summ, W, steps)
    kern = kernel_times(torch, summ, W)
    gaps = timeline_gaps(torch, summ, W, trace_path=trace)
    from traceml_b200 import _abi

    stream = ("packed" if _abi.lib().tml_ring_packed_(eng.handle, W) == 1 else
              "certified" if _abi.lib().tml_ring_certified_(eng.handle, W) == 1 else "general")
    eng.close()
    del host, recs
    med = {k: statistics.median(v) for k, v in stage.items() if not k.startswith("host_")}
    wall_ms, sj_ms = statistics.median(wall), statistics.median(sj)
    ceil = copy_ceiling(torch)
    # bytes read per step by the stream that ran, plus 8 series x 8 B written when the pairs are
    # mapped twice (series_paired), 16 x 8 B otherwise
    fused_bytes = W * ({"packed": 32.0, "certified": 64.0, "general": 65.0}[stream] + (64.0 if paired else 128.0))
    k3a = med.get("k3a") or 0.0
    fused_gbps = fused_bytes / (k3a * 1e-3) / 1e9 if k3a else None
    return {
        "window": W, "steps": steps, "fused_rows": fused, "series_paired": paired, "stream": stream,
        "build_ms": build_ms, "build_wall_ms": wall_ms, "launches_per_build": launches,
        "stage_ms": med, "sections_json_ms": sj_ms,
        "python_rest_ms": wall_ms - med.get("total", 0.0) - sj_ms,
        "native_minus_fused_ms": med.get("total", 0.0) - k3a,
        "segments_ms": seg, "kernel_ms": kern,
        # what the device does not spend in the pass or the band sums (both timed on the device)
        "device_idle_ms": build_ms - k3a - (kern.get("k_bands") or 0.0),
        "timeline_ms": gaps,
        "copy_ceiling": ceil,
        "fused_pass": {"bytes": fused_bytes, "ms": k3a, "GBps": fused_gbps,
                       "of_copy_ceiling": (fused_gbps / ceil["GBps"]) if fused_gbps else None,
                       "of_datasheet_3350": (fused_gbps / 3350.0) if fused_gbps else None},
        "gpu": gpu_info(0),
    }


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=1000, help="K: builds per timed loop")
    ap.add_argument("--window", type=int, default=4_000_000, help="W: step records")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--trace", default="", help="also write the timeline's Chrome trace to this path")
    args = ap.parse_args()
    if args.steps < 1 or args.window < 1:
        ap.error("--steps and --window must be at least 1")
    print(json.dumps(measure(args.steps, args.window, args.warmup, args.trace)), flush=True)


if __name__ == "__main__":
    main()
