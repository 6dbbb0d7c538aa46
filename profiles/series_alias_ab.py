"""A/B of the single-rank build's paired series against the plain 16-row series buffer.

With one rank the bulk build stores each median / worst series pair once and maps it at both rows
(``TML_SERIES_ALIAS=1``, the default); ``TML_SERIES_ALIAS=0`` keeps the plain buffer with all 16 rows
written.  Both arms run the same workload in child processes, alternating over ``--rounds`` rounds
(the arm that goes first alternates too), each round running ``profiles/single_rank_build.py`` and
``bench.py --gpus 1`` once per arm.  Prints one JSON line per round as it finishes, then one with
everything:

  * ``rounds``: per round and arm, ``build_ms`` / ``pass_ms`` / ``device_idle_ms`` /
    ``launches_per_build`` (single_rank_build.py) and ``ms_per_step`` / ``sustained_ms`` / parity
    (bench.py);
  * ``arms``: median, min and max of each timing per arm, and the pass's physical bytes against the
    measured device-to-device copy ceiling;
  * ``ms_per_step_drop``: 1 - median(paired) / median(plain), and whether the two ranges overlap;
  * ``dumps_identical``: every bench run's ``--dump-outputs`` files, byte for byte, against the first;
  * ``gpu``: card name, power limit and max SM clock (read-only ``nvidia-smi`` query).

Dumps go to a temporary directory, so the tree can stay read-only.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from single_rank_build import gpu_info  # noqa: E402

ARMS = ("0", "1")  # TML_SERIES_ALIAS: plain, paired


def child(cmd, alias: str) -> dict:
    env = dict(os.environ, TML_SERIES_ALIAS=alias)
    p = subprocess.run([sys.executable] + cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3600)
    lines = [x for x in p.stdout.splitlines() if x.startswith("{")]
    if p.returncode != 0 or not lines:
        raise RuntimeError(f"{cmd[0]} (TML_SERIES_ALIAS={alias}) exited {p.returncode}: {p.stderr[-2000:]}")
    return json.loads(lines[-1])


def same_files(a: str, b: str) -> bool:
    names = sorted(os.listdir(a))
    if not names or names != sorted(os.listdir(b)):
        return False
    for name in names:
        with open(os.path.join(a, name), "rb") as fa, open(os.path.join(b, name), "rb") as fb:
            if fa.read() != fb.read():
                return False
    return True


def spread(v) -> dict:
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=int, default=4_000_000, help="W: step records")
    ap.add_argument("--build-steps", type=int, default=300, help="builds per timed loop of single_rank_build.py")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=5)
    args = ap.parse_args()
    if args.rounds < 1:
        ap.error("--rounds must be at least 1")
    gpu = gpu_info(0)
    rounds, dumps = [], []
    with tempfile.TemporaryDirectory(prefix="tml_alias_ab_") as tmp:
        for rnd in range(args.rounds):
            row = {}
            for alias in (ARMS if rnd % 2 == 0 else ARMS[::-1]):
                b = child(["profiles/single_rank_build.py", "--window", str(args.window),
                           "--steps", str(args.build_steps)], alias)
                d = os.path.join(tmp, f"alias{alias}_round{rnd}")
                m = child(["bench.py", "--gpus", "1", "--window", str(args.window), "--steps", str(args.bench_steps),
                           "--warmup", str(args.bench_warmup), "--no-overhead", "--no-cpu-baseline",
                           "--dump-outputs", d], alias)
                dumps.append(d)
                par = m.get("parity") or {}
                row[alias] = {
                    "series_paired": b["series_paired"], "build_ms": b["build_ms"],
                    "pass_ms": b["fused_pass"]["ms"], "pass_bytes": b["fused_pass"]["bytes"],
                    "device_idle_ms": b["device_idle_ms"], "launches_per_build": b["launches_per_build"],
                    "copy_ceiling_GBps": b["copy_ceiling"]["GBps"],
                    "ms_per_step": m["ms_per_step"], "sustained_ms": m["sustained"]["ms_per_step"],
                    "value": m["value"], "gpu_launches": m["gpu_launches"],
                    "parity_ok": par.get("ok"), "series_bit_equal": (par.get("series") or {}).get("bit_equal"),
                }
            rounds.append(row)
            print(json.dumps({"round": rnd, **{("paired" if a == "1" else "plain"): v for a, v in row.items()}}),
                  flush=True)
        dumps_identical = all(same_files(dumps[0], d) for d in dumps[1:])
    arms = {}
    for alias in ARMS:
        rs = [r[alias] for r in rounds]
        pass_ms = statistics.median(r["pass_ms"] for r in rs)
        ceil = statistics.median(r["copy_ceiling_GBps"] for r in rs)
        gbps = rs[0]["pass_bytes"] / (pass_ms * 1e-3) / 1e9
        arms["paired" if alias == "1" else "plain"] = {
            **{k: spread([r[k] for r in rs]) for k in ("ms_per_step", "sustained_ms", "build_ms", "pass_ms",
                                                      "device_idle_ms")},
            "series_paired": [r["series_paired"] for r in rs],
            "launches_per_build": [r["launches_per_build"] for r in rs],
            "parity_ok": all(r["parity_ok"] for r in rs), "series_bit_equal": all(r["series_bit_equal"] for r in rs),
            "pass": {"bytes": rs[0]["pass_bytes"], "GBps": gbps, "copy_ceiling_GBps": ceil, "of_copy_ceiling": gbps / ceil},
        }
    plain, paired = arms["plain"]["ms_per_step"], arms["paired"]["ms_per_step"]
    print(json.dumps({
        "window": args.window, "rounds": rounds, "arms": arms,
        "ms_per_step_drop": 1.0 - paired["median"] / plain["median"],
        "ranges_overlap": paired["max"] >= plain["min"],
        "dumps_identical": dumps_identical, "gpu": gpu, "gpu_after": gpu_info(0),
    }), flush=True)


if __name__ == "__main__":
    main()
