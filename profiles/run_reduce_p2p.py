"""Workload for an ncu capture of K4 under REAL peer loads: torchrun, one rank per GPU, every rank
holds W step records, the native driver reduces with the fused NVLink peer-load exchange ("p2p").
Launch it under torchrun with the profiler wrapping rank 0 only.
Usage: ... profiles/run_reduce_p2p.py [W] [reps]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import replay  # noqa: E402
from traceml_b200 import sections  # noqa: E402
from traceml_b200.engine import Engine  # noqa: E402
from traceml_b200.reduce import TorchDistComm  # noqa: E402

W = int(sys.argv[1]) if len(sys.argv) > 1 else 4_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
recs = replay.make_step_replay("balanced", world, W, seed=1, only_ranks=[rank])[rank]
e = Engine(device=local, rank=rank, world=world, ring_slots=W, proc_slots=65536)
e.load_steps(recs)
e.load_procs(replay.make_proc_replay("normal", world, 60000, seed=1, only_ranks=[rank])[rank])
torch.cuda.synchronize()
summ = sections.SummaryEngine([e], TorchDistComm(), exchange="p2p", ram_total=replay.PROC_RAM_TOTAL_BYTES,
                              gpu_count=world)
import re
import subprocess
import time


def nvlink_kib(idx):
    """Cumulative NVLink data counters of one GPU (nvidia-smi nvlink -gt d): (tx KiB, rx KiB) over all links."""
    try:
        txt = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", str(idx)], capture_output=True, text=True,
                             timeout=30).stdout
        tx = sum(int(v) for v in re.findall(r"Data Tx:\s*(\d+)\s*KiB", txt))
        rx = sum(int(v) for v in re.findall(r"Data Rx:\s*(\d+)\s*KiB", txt))
        return tx, rx, txt[:400]
    except Exception as exc:  # noqa: BLE001
        return None, None, str(exc)


for _ in range(3):
    out = summ.build(W, 60000)
torch.cuda.synchronize()
dist.barrier()
before = nvlink_kib(local) if rank == 0 else None
dist.barrier()
t0 = time.perf_counter()
k4 = []
for _ in range(reps):
    out = summ.build(W, 60000)
    k4.append(out["reduce"].timings_ms.get("k4"))
torch.cuda.synchronize()
dt = time.perf_counter() - t0
dist.barrier()
if rank == 0:
    after = nvlink_kib(local)
    n_shard = W // world
    expect = (world - 1) * n_shard * 64
    line = {"ranks": world, "window": W, "reps": reps, "ms_per_reduce": dt / reps * 1e3,
            "k4_ms_median": sorted(k4)[len(k4) // 2], "exchange": out["reduce"].exchange,
            "expected_peer_row_bytes_in_per_reduce": expect}
    if before[0] is not None and after[0] is not None:
        line["nvlink_rx_bytes_per_reduce"] = (after[1] - before[1]) * 1024 / reps
        line["nvlink_tx_bytes_per_reduce"] = (after[0] - before[0]) * 1024 / reps
        line["rx_over_expected"] = line["nvlink_rx_bytes_per_reduce"] / expect
        if line["k4_ms_median"]:
            line["rx_GBps_during_k4"] = expect / (line["k4_ms_median"] * 1e-3) / 1e9
    else:
        line["nvlink_counters"] = "unavailable: " + str(before[2])[:200]
    import json
    print(json.dumps(line))
    print("ok", out["step_time"]["diagnosis"]["primary"]["status"], out["reduce"].exchange, out["reduce"].timings_ms)
dist.barrier()
e.close()
dist.destroy_process_group()
