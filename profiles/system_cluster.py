"""What the multi-node System section adds on comm index 0's device, apart from the gather.

Prints one JSON line:

  * ``gpu``: card name, power limit and max SM clock (read-only ``nvidia-smi`` query);
  * ``pack_ms``: device time of one ``tml_sys_node_pack`` (the record assembled in HBM from the
    node's K6s result), CUDA events around each of ``--reps`` launches after warm-up;
  * ``cluster_ms[n]``: device time of ``tml_sys_cluster_launch`` over n = 2, 8, 64 gathered records
    (K6m plus the one device-to-host copy of the records and the cluster rollup), the same way.
    Each record comes from a node of 10^3 samples of 8 GPUs.

The all-gather between hosts is not measured: it needs several hosts.

    python profiles/system_cluster.py [--reps 200]
"""
from __future__ import annotations

import argparse
import ctypes as C
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


def _timed(torch, stream, fn, reps):
    ms = []
    for i in range(reps + 10):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            a.record()
            fn()
            b.record()
        b.synchronize()
        if i >= 10:
            ms.append(a.elapsed_time(b))
    return _stats(ms)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    import torch

    import system_cases as sc
    import system_cluster_cases as scc
    from single_rank_build import gpu_info
    from traceml_b200 import _abi, sections
    from traceml_b200.engine import Engine

    torch.cuda.set_device(0)
    s = torch.cuda.Stream()
    sp = int(s.cuda_stream)
    rec = C.sizeof(_abi.SysNodeRecord)
    eng = Engine(device=0, rank=0, world=1, ring_slots=1024, proc_slots=1_000)
    eng.load_sys(sc.sys_records(sc.random_raw(1_000, 8, seed=1)), sp)
    eng.sys_reduce_launch(1_000, sp)
    eng.sys_reduce_collect()
    n_max = 64
    buf = torch.empty(n_max * rec + C.sizeof(_abi.SysClusterOut), dtype=torch.uint8, device="cuda")
    idents = [sections.node_ident(scc.identity(k, n_max)) for k in range(n_max)]
    pack = _timed(torch, s, lambda: eng.sys_node_pack(idents[0], buf, sp), args.reps)
    cluster = {}
    for n in (2, 8, 64):
        for k in range(n_max):  # distinct node labels, so K6m folds every record; the result of a
            eng.sys_node_pack(idents[k], buf[k * rec:], sp)  # smaller n lands on records n, n + 1
        ms = _timed(torch, s, lambda: eng.sys_cluster_launch(buf, n, sp), args.reps)
        records, out = eng.sys_cluster_collect(n)
        assert out.n_nodes == n and out.agg.n == n * 1_000
        cluster[str(n)] = ms
    eng.close()
    print(json.dumps({"gpu": gpu_info(0), "pack_ms": pack, "cluster_ms": cluster}))


if __name__ == "__main__":
    main()
