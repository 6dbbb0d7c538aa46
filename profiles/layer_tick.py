"""Time one tick of the live layer-time panel: ``live.LayerCombinedTimerData`` (device stages on its
side stream) against the unmodified reference ``LayerCombinedTimerData.compute_display_data()``
(Python over wire rows), on the same records.

Models of 64 / 256 / 1024 layers, a ring of 256 steps, R = 1 and R = 4 ranks (R > 1 played by
several engines in one process).  Each configuration runs 5 alternating rounds of (twin tick,
reference tick); reported: median (min-max) in ms of
  twin_tick_ms    host clock around the whole tick, after a device synchronise
  twin_device_ms  CUDA events on the tick's stream around the same tick
  ref_tick_ms     host clock around the reference's tick
The card's name, power limit and max SM clock are printed with the numbers.

    python profiles/layer_tick.py [--rounds 5] [--ring 256]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as exc:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "error": str(exc)}


def spread(xs) -> str:
    return f"{statistics.median(xs):.3f} ({min(xs):.3f}-{max(xs):.3f})"


def run(n_layers: int, R: int, ring: int, rounds: int) -> dict:
    import layer_tick_cases as ltc
    from traceml_b200 import _abi
    from traceml_b200.engine import Engine
    from traceml_b200.instrumentation.layers import LayerProfile
    from traceml_b200.live import LayerCombinedTimerData

    rng = np.random.default_rng(n_layers * 10 + R)
    recs = {r: ltc.make_records(list(range(1, ring + 1 - r)), n_layers, rng) for r in range(R)}
    engines = [Engine(device=0, rank=r, world=R, ring_slots=64, proc_slots=64) for r in range(R)]
    models = [torch.nn.Sequential(*[torch.nn.Identity() for _ in range(n_layers)]) for _ in range(R)]
    profiles = [LayerProfile(e, m, ring_steps=ring) for e, m in zip(engines, models)]
    for p, r in zip(profiles, range(R)):
        a = np.ascontiguousarray(recs[r])
        _abi.check(_abi.lib().tml_layer_load_(p.engine._h, a.ctypes.data, len(a), None), "tml_layer_load_")
    names = profiles[0].names
    twin = LayerCombinedTimerData(profiles)
    ref_mod = __import__("traceml.renderers.layer_combined_time.compute", fromlist=["x"])
    ref_mod.get_ddp_info = lambda: (R > 1, 0, R)
    ref = ref_mod.LayerCombinedTimerData(remote_store=ltc.reference_store(recs, names))
    twin.compute_display_data()  # warm: modules, workspaces, identity exchange
    ref.compute_display_data()
    t_twin, t_dev, t_ref = [], [], []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(twin._stream)
        t0 = time.perf_counter()
        got = twin.compute_display_data()
        t_twin.append((time.perf_counter() - t0) * 1e3)
        e1.record(twin._stream)
        e1.synchronize()
        t_dev.append(e0.elapsed_time(e1))
        t0 = time.perf_counter()
        ref.compute_display_data()
        t_ref.append((time.perf_counter() - t0) * 1e3)
    assert got["safe_step"] == ring - R + 1 and len(got["all_items"]) == n_layers, got["status_message"]
    for p in profiles:
        p.detach()
    for e in engines:
        e.close()
    return {"n_layers": n_layers, "ranks": R, "ring_steps": ring, "rounds": rounds,
            "twin_tick_ms": spread(t_twin), "twin_device_ms": spread(t_dev), "ref_tick_ms": spread(t_ref),
            "speedup_median": round(statistics.median(t_ref) / statistics.median(t_twin), 1)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ring", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profiles/layer_tick.py measures on a CUDA device; none found")
    import layer_tick_cases as ltc

    if not ltc.reference_importable():
        sys.exit("the reference is not installed in oracle/_ref (build() installs it)")
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}))
    for n_layers in (64, 256, 1024):
        for R in (1, 4):
            print(json.dumps(run(n_layers, R, args.ring, args.rounds)))


if __name__ == "__main__":
    main()
