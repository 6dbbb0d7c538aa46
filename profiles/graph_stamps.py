"""Device cost of ``trace_graph``: a whole training step captured in a CUDA graph, with and without
its regions' stamps (forward, backward, optimizer: six 1-warp kernel nodes per replay).

Workloads: bench.py's micro-MLP (Linear 8x8, batch 16) and BASELINE config 2 (synthetic ResNet-18,
batch 64x3x224x224), each with capturable Adam.  Per workload two graphs of the same step are
captured from two identical copies of the model, one inside ``trace_graph``.  After warm-up, each
of ``--rounds`` rounds (the arm that goes first alternates) times ``--replays`` back-to-back
``g.replay()`` per arm with CUDA events; the per-replay time is the pair's elapsed time over the
replays.  Prints one JSON line: per workload and arm the median / min / max over rounds, the
per-round difference stamped - plain (median and spread), and the card's name and power limit.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import torch  # noqa: E402

from single_rank_build import gpu_info  # noqa: E402


def capture(model, x, y, stamped: bool):
    import traceml_b200 as traceml

    opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(x), y).backward()
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    opt.zero_grad(set_to_none=True)
    g = torch.cuda.CUDAGraph()
    if stamped:
        with traceml.trace_graph(model), torch.cuda.graph(g):
            torch.nn.functional.cross_entropy(model(x), y).backward()
            opt.step()
    else:
        with torch.cuda.graph(g):
            torch.nn.functional.cross_entropy(model(x), y).backward()
            opt.step()
    return g, opt


def per_replay_us(g, n: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / n


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def run(name, model, x, y, replays: int, rounds: int) -> dict:
    from traceml_b200 import runtime

    graphs = {"plain": capture(copy.deepcopy(model), x, y, False),
              "stamped": capture(copy.deepcopy(model), x, y, True)}
    for g, _ in graphs.values():
        per_replay_us(g, max(10, replays // 4))  # warm-up
    runtime.get_engine().reset()
    res = {"plain": [], "stamped": []}
    for r in range(rounds):
        for arm in (("plain", "stamped") if r % 2 == 0 else ("stamped", "plain")):
            res[arm].append(per_replay_us(graphs[arm][0], replays))
    recs, _ = runtime.get_engine().drain()  # nothing is committed: the stamps sit in the open step
    diff = [s - p for s, p in zip(res["stamped"], res["plain"])]
    return {"workload": name, "replays_per_round": replays, "rounds": rounds,
            "plain_us": spread(res["plain"]), "stamped_us": spread(res["stamped"]),
            "added_us": spread(diff), "added_pct_of_plain": 100.0 * statistics.median(diff) / statistics.median(res["plain"]),
            "per_round": res, "records_committed": len(recs)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mlp-replays", type=int, default=2000)
    ap.add_argument("--resnet-replays", type=int, default=60)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_stamps.py measures on the GPU: no CUDA device")
    import traceml_b200 as traceml
    from bench import resnet18

    torch.cuda.set_device(0)
    traceml.init(mode="auto")
    torch.manual_seed(0)
    out = {"gpu": gpu_info(0), "results": []}
    mlp = torch.nn.Linear(8, 8).cuda()
    out["results"].append(run("micro_mlp", mlp, torch.randn(16, 8, device="cuda"),
                              torch.randint(0, 8, (16,), device="cuda"), a.mlp_replays, a.rounds))
    net = resnet18().cuda()
    out["results"].append(run("resnet18_b64", net, torch.randn(64, 3, 224, 224, device="cuda"),
                              torch.randint(0, 10, (64,), device="cuda"), a.resnet_replays, a.rounds))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
