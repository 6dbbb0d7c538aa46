"""Device time of one step-ring load: ``load_steps_ptr`` of the bench's W records from pinned memory.

Loads the replay ``bench.py --gpus 1`` builds from (``balanced``, seed 1, ``Engine(ring_slots=W)``)
``--reps`` times into the same ring, CUDA events around each load on the caller's stream, and prints
one JSON line with the median, min and max in ms.  ``--tree`` imports the package from another built
tree, so that two trees' loads can be timed alternately by the same script.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--tree", default=ROOT, help="built tree whose package is timed (default: this tree)")
    ap.add_argument("--window", type=int, default=4_000_000, help="W: step records")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    sys.path.insert(0, tree)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch

    import replay
    from traceml_b200.engine import Engine

    assert torch.cuda.is_available(), "ring_load.py needs a CUDA device"
    torch.cuda.set_device(0)
    W = int(args.window)
    recs = replay.make_step_replay("balanced", 1, W, seed=1, only_ranks=[0])[0]
    host = torch.empty(W * 128, dtype=torch.uint8).pin_memory()
    host.numpy()[:] = recs.view(np.uint8).reshape(-1)
    eng = Engine(device=0, rank=0, world=1, ring_slots=W, proc_slots=64)
    stream = torch.cuda.current_stream()
    eng.load_steps_ptr(host.data_ptr(), W, stream.cuda_stream)  # warm-up: staging buffers, streams
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.load_steps_ptr(host.data_ptr(), W, stream.cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    eng.close()
    print(json.dumps({"tree": tree, "window": W, "load_ms": {"median": statistics.median(ms), "min": min(ms),
                                                              "max": max(ms), "all": ms}}), flush=True)


if __name__ == "__main__":
    main()
