"""What the System section costs on the device, and whether it hides under the window pass.

Prints one JSON line:

  * ``gpu``: card name, power limit and max SM clock (read-only ``nvidia-smi`` query);
  * ``k_sys_reduce_ms``: device time of K6s alone (CUDA events around ``tml_sys_reduce_launch`` on a
    stream of its own), G = 8 GPUs per sample, at n = 10^3, 10^4, 10^5 samples: median, min, max of
    ``--reps`` launches after warm-up;
  * ``build``: the single-rank build at W = 4e6 steps (the ``bench.py --gpus 1`` workload shape: dense
    balanced replay, 60 000 process samples), with 10^4 system samples against none, ``--rounds``
    alternating rounds of ``--builds`` back-to-back builds each.  ``build_ms`` is CUDA events around
    each ``SummaryEngine.build`` (it ends in the build's own wait), per arm: median and min-max of the
    per-round medians; ``extra_ms`` = with minus without.

    python profiles/system_section.py [--window 4000000] [--rounds 5] [--builds 20] [--reps 50]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))


def _stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def kernel_times(torch, reps: int) -> dict:
    import system_cases as sc
    from traceml_b200.engine import Engine

    out = {}
    for n in (1_000, 10_000, 100_000):
        eng = Engine(device=0, rank=0, world=1, ring_slots=1024, proc_slots=n)
        eng.load_sys(sc.sys_records(sc.random_raw(n, 8, seed=n)))
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        ms = []
        for i in range(reps + 5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s):
                a.record()
                eng.sys_reduce_launch(n, int(s.cuda_stream))
                b.record()
            eng.sys_reduce_collect()
            b.synchronize()
            if i >= 5:
                ms.append(a.elapsed_time(b))
        out[str(n)] = _stats(ms)
        eng.close()
    return out


def build_times(torch, window: int, rounds: int, builds: int) -> dict:
    import numpy as np

    import replay
    import system_cases as sc
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    recs = np.ascontiguousarray(replay.make_step_replay("balanced", 1, window, seed=0)[0])
    procs = replay.make_proc_replay("normal", 1, 60_000, seed=0)[0]
    arms = {}
    for name, with_sys in (("none", False), ("with_10k_samples", True)):
        eng = Engine(device=0, rank=0, world=1, ring_slots=window, proc_slots=65_536)
        eng.load_steps(recs)
        eng.load_procs(procs)
        if with_sys:
            eng.load_sys(sc.sys_records(sc.random_raw(10_000, 8, seed=1)))
        torch.cuda.synchronize()
        se = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1,
                                    system_identity=sc.IDENTITY)
        for _ in range(3):
            se.build(window, 10_000)
        arms[name] = (eng, se)
    per_round = {k: [] for k in arms}
    launches = {}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(list(arms)))
        for name in order:
            eng, se = arms[name]
            ms = []
            l0 = eng.launch_count
            for _ in range(builds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                res = se.build(window, 10_000)
                b.record()
                b.synchronize()
                ms.append(a.elapsed_time(b))
            launches[name] = (eng.launch_count - l0) / builds
            assert res["system"]["diagnosis"]["primary"]["kind"] != ("NO_DATA" if name != "none" else None)
            per_round[name].append(statistics.median(ms))
    out = {k: dict(_stats(v), rounds=v, launches_per_build=launches[k]) for k, v in per_round.items()}
    out["extra_ms"] = out["with_10k_samples"]["median"] - out["none"]["median"]
    for eng, _ in arms.values():
        eng.close()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=int, default=4_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--builds", type=int, default=20)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch

    from single_rank_build import gpu_info

    torch.cuda.set_device(0)
    print(json.dumps({"gpu": gpu_info(0), "k_sys_reduce_ms": kernel_times(torch, args.reps),
                      "build": build_times(torch, args.window, args.rounds, args.builds)}))


if __name__ == "__main__":
    main()
