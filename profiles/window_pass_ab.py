"""A/B of the single-rank window pass's tile loops between two built source trees on one GPU.

``bench.py`` runs only the packed stream of ``k_window_fused``.  This script times every loop of the
pass on seeded rings of W records (``Engine(ring_slots=W)``, one load), each tree in a process of its
own, alternating the trees (and which goes first) over ``--rounds`` rounds:

  * ``fused_packed``: dense records inside the packed ranges (``test_gpu_packed_ring._recs``), so the
    window is certified and packed-streamable: the packed stream;
  * ``fused_hot``: the same records with one too wide for its packed copy: the hot-half stream;
  * ``fused_general``: the same records with one step id skipped: the general loop;
  * ``rows_W`` / ``rows_131072``: ``k_window_rows`` (``tml_win_prepare``) on the ``fused_general`` ring
    at window W, and at 2^17, where it also adds up the chunk sums of the reference-order sums.

Each time is the median of ``kernel_ms(0)`` (the library's events around the pass) over ``--passes``
calls after ``--warmup``.  Prints one JSON line: per tree and loop the median, min and max over the
rounds, whether each loop's range overlaps tree A's, whether the returned ``WinInfo`` / ``AlignInfo``
structs (their ``kernel_ms`` zeroed) and a checksum of the fused series are identical across trees and
rounds, and the card's name, power limit and max SM clock (read-only ``nvidia-smi`` query).
Both trees must already be built (``__graft_entry__.build()``); tree A is usually the parent commit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from single_rank_build import gpu_info  # noqa: E402


def rings(W: int, seed: int) -> dict:
    import test_gpu_packed_ring as pk

    packed = pk._recs(W, seed)
    general = packed.copy()
    general["step"][W // 2:] += 1
    return {"packed": packed, "hot": pk._wide(packed, [W // 2]), "general": general}


def child(tree: str, W: int, seed: int, passes: int, warmup: int) -> dict:
    sys.path.insert(0, tree)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch

    from traceml_b200 import _abi
    from traceml_b200.engine import Engine

    assert torch.cuda.is_available(), "window_pass_ab.py needs a CUDA device"
    torch.cuda.set_device(0)
    lib, out = _abi.lib(), {}

    def timed(eng, call):
        for _ in range(warmup):
            call()
        ms = []
        for _ in range(passes):
            digest = call()
            ms.append(eng.kernel_ms(0))
        return {"ms": statistics.median(ms), "out": hashlib.sha256(digest).hexdigest()[:16]}

    for name, recs in rings(W, seed).items():
        eng = Engine(device=0, rank=0, world=1, ring_slots=W, proc_slots=64)
        eng.load_steps(recs)
        torch.cuda.synchronize()
        buf = torch.zeros(16 * W, dtype=torch.float64, device="cuda")
        info, al, ok = _abi.WinInfo(), _abi.AlignInfo(), C.c_uint32(0)

        def fused():
            _abi.check(lib.tml_win_fused(eng.handle, W, buf.data_ptr(), 0, C.byref(info), C.byref(al), C.byref(ok)),
                       "tml_win_fused")
            info.kernel_ms = 0.0
            return bytes(info) + bytes(al) + bytes(ok) + buf.view(torch.int64).sum().cpu().numpy().tobytes()

        def prepare(window):
            got = eng.win_prepare(window)
            got.kernel_ms = 0.0
            return bytes(got)

        out[f"fused_{name}"] = timed(eng, fused)
        if name == "general":
            for window in (W, 1 << 17):
                out[f"rows_{window}"] = timed(eng, lambda: prepare(window))
        del buf
        eng.close()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--a", help="tree A (the parent)")
    ap.add_argument("--b", default=ROOT, help="tree B (default: this tree)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=int, default=4_000_000, help="W: step records")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--passes", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--child", help=argparse.SUPPRESS)  # a tree to measure in this process
    args = ap.parse_args()
    knobs = [str(x) for x in (args.window, args.seed, args.passes, args.warmup)]
    if args.child:
        print(json.dumps(child(args.child, *map(int, knobs))), flush=True)
        return
    if not args.a:
        ap.error("--a is required")
    trees = {"A": os.path.abspath(args.a), "B": os.path.abspath(args.b)}
    runs = {"A": [], "B": []}
    for r in range(args.rounds):
        for name in ("A", "B") if r % 2 == 0 else ("B", "A"):
            tree = trees[name]
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", tree, "--window", knobs[0],
                                "--seed", knobs[1], "--passes", knobs[2], "--warmup", knobs[3]],
                               capture_output=True, text=True, timeout=1800)
            lines = [x for x in p.stdout.splitlines() if x.startswith("{")]
            if p.returncode != 0 or not lines:
                raise RuntimeError(f"tree {name} round {r} exited {p.returncode}: {p.stderr[-2000:]}")
            runs[name].append(json.loads(lines[-1]))
            print(json.dumps({"round": r, "tree": name, **{k: v["ms"] for k, v in runs[name][-1].items()}}),
                  file=sys.stderr, flush=True)
    report = {"gpu": gpu_info(0), "trees": trees, "rounds": args.rounds, "window": args.window, "loops": {}}
    for loop in runs["A"][0]:
        row = {}
        for name in trees:
            v = [x[loop]["ms"] for x in runs[name]]
            row[name] = {"median": statistics.median(v), "min": min(v), "max": max(v), "all": v}
        row["ranges_overlap"] = row["B"]["min"] <= row["A"]["max"] and row["A"]["min"] <= row["B"]["max"]
        row["outputs_identical"] = len({x[loop]["out"] for n in trees for x in runs[n]}) == 1
        report["loops"][loop] = row
    report["all_identical"] = all(v["outputs_identical"] for v in report["loops"].values())
    print(json.dumps(report), flush=True)


if __name__ == "__main__":
    main()
