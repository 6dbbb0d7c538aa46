"""A/B of two built source trees on one GPU: ``bench.py --gpus 1`` alternated between them.

Runs ``bench.py --gpus 1 --steps K --warmup W --no-cpu-baseline`` from tree A, then from tree B, for
``--rounds`` rounds, each in a process of its own, and prints one JSON line with, per tree, the median
and min-max of: ``ms_per_step``, ``sustained.ms_per_step``, the fused pass
(``roofline.kernels.k_window_fused.ms``), ``e2e.ms_per_step``, ``default_window.ms`` and
``step_overhead.micro_mlp.b200_overhead_us``, the step path's ``step_overhead.telemetry_rate.step_records_per_s``
and ``step_overhead.api_cost_us.step_commit``, and the device time of one ring load of the bench's
records (``profiles/ring_load.py`` of this tree run against each tree, once per round, median of its
loads); plus ``parity.ok`` / ``series.bit_equal`` of every run,
whether the ``--dump-outputs`` files of the first round are byte-identical between the trees,
``profiles/single_rank_build.py``'s pass-vs-copy-ceiling figures, device idle time, timeline gaps and
host segments of each tree (one run each, after the rounds) and the card's name, power limit and max SM clock (read-only ``nvidia-smi`` query).

Both trees must already be built (``__graft_entry__.build()``).  Tree A is usually the parent commit
and tree B the change under test: any two trees whose bench and profile take these arguments.
"""
from __future__ import annotations

import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from single_rank_build import gpu_info  # noqa: E402

METRICS = {
    "ms_per_step": ("ms_per_step",),
    "sustained_ms_per_step": ("sustained", "ms_per_step"),
    "fused_pass_ms": ("roofline", "kernels", "k_window_fused", "ms"),
    "e2e_ms_per_step": ("e2e", "ms_per_step"),
    "default_window_ms": ("default_window", "ms"),
    "micro_mlp_overhead_us": ("step_overhead", "micro_mlp", "b200_overhead_us"),
    "step_records_per_s": ("step_overhead", "telemetry_rate", "step_records_per_s"),
    "step_commit_us": ("step_overhead", "api_cost_us", "step_commit"),
    "ring_load_ms": ("ring_load", "load_ms", "median"),
}


def dig(d, path):
    for k in path:
        if not isinstance(d, dict) or k not in d:
            return None
        d = d[k]
    return d


def last_json(text: str) -> dict:
    for line in reversed(text.strip().splitlines()):
        line = line.strip()
        if line.startswith("{"):
            try:
                return json.loads(line)
            except json.JSONDecodeError:
                continue
    return {}


def run(tree: str, args: list, timeout: int = 1800) -> dict:
    p = subprocess.run([sys.executable] + args, cwd=tree, capture_output=True, text=True, timeout=timeout)
    out = last_json(p.stdout)
    if p.returncode != 0 or not out:
        out.setdefault("error", f"rc={p.returncode}: " + (p.stderr or p.stdout)[-600:])
    return out


def summary(values):
    v = [x for x in values if x is not None]
    if not v:
        return None
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "n": len(v), "all": v}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--a", required=True, help="tree A (the parent)")
    ap.add_argument("--b", default=ROOT, help="tree B (default: this tree)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", required=True, help="directory for the dumped outputs and the raw runs")
    ap.add_argument("--no-overhead", action="store_true",
                    help="pass --no-overhead to bench.py: skip the step-overhead leg (its metrics stay empty)")
    args = ap.parse_args()
    trees = {"A": os.path.abspath(args.a), "B": os.path.abspath(args.b)}
    os.makedirs(args.out, exist_ok=True)
    runs = {"A": [], "B": []}
    for r in range(args.rounds):
        for name, tree in trees.items():
            cmd = [os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
                   "--warmup", str(args.warmup), "--no-cpu-baseline"] + (["--no-overhead"] if args.no_overhead else [])
            if r == 0:
                cmd += ["--dump-outputs", os.path.join(os.path.abspath(args.out), f"dump_{name}")]
            res = run(tree, cmd)
            res["ring_load"] = run(tree, [os.path.join(ROOT, "profiles", "ring_load.py"), "--tree", tree])
            runs[name].append(res)
            print(json.dumps({"round": r, "tree": name, **{k: dig(res, p) for k, p in METRICS.items()},
                              "error": res.get("error")}), file=sys.stderr, flush=True)
    with open(os.path.join(args.out, "runs.json"), "w") as fh:
        json.dump(runs, fh)
    report = {"gpu": gpu_info(0), "trees": trees, "rounds": args.rounds, "steps": args.steps}
    for name in trees:
        report[name] = {k: summary([dig(x, p) for x in runs[name]]) for k, p in METRICS.items()}
        report[name]["parity_ok"] = [dig(x, ("parity", "ok")) for x in runs[name]]
        report[name]["series_bit_equal"] = [dig(x, ("parity", "series", "bit_equal")) for x in runs[name]]
    da, db = (os.path.join(args.out, f"dump_{n}") for n in ("A", "B"))
    files = sorted(os.listdir(da)) if os.path.isdir(da) else []
    report["dump_identical"] = bool(files) and files == sorted(os.listdir(db)) and all(
        filecmp.cmp(os.path.join(da, f), os.path.join(db, f), shallow=False) for f in files)
    for name, tree in trees.items():
        srb = run(tree, [os.path.join(tree, "profiles", "single_rank_build.py"), "--steps", "300"])
        report[name]["single_rank_build"] = {"fused_pass": srb.get("fused_pass"),
                                             "copy_ceiling": srb.get("copy_ceiling"),
                                             "build_ms": srb.get("build_ms"), "device_idle_ms": srb.get("device_idle_ms"),
                                             "timeline_ms": srb.get("timeline_ms"), "segments_ms": srb.get("segments_ms"),
                                             "error": srb.get("error")}
    print(json.dumps(report), flush=True)


if __name__ == "__main__":
    main()
