"""Cost of captured steps: a training step captured in a CUDA graph with its ``trace_step`` inside the
capture (a captured begin stamp and commit per replay) against the same step captured with its
regions' stamps only (``trace_graph`` alone).

Workloads: bench.py's micro-MLP (Linear 8x8, batch 16) and BASELINE config 2 (synthetic ResNet-18,
batch 64x3x224x224), each with capturable Adam, as profiles/graph_stamps.py.

Device time: per workload both graphs are captured from two identical copies of the model; each of
``--rounds`` rounds (the arm that goes first alternates) times ``--replays`` back-to-back
``g.replay()`` per arm with CUDA events.  Host time (micro-MLP): the host's time per iteration of
``for ...: g.replay()`` over the captured-step graph against ``with trace_step(model): g.replay()``
over the stamps-only graph, each loop ended by one synchronise.  The second loop runs first, on an
engine that has not entered device-committed mode, so it measures today's path; the rounds of the
host comparison therefore do not alternate.  Prints one JSON line with the card's name and power
limit.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import torch  # noqa: E402

from graph_stamps import per_replay_us, spread  # noqa: E402
from single_rank_build import gpu_info  # noqa: E402


def capture(model, x, y, steps: bool):
    """The step in a graph, inside trace_graph; `steps`: with its trace_step captured too."""
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
    with traceml.trace_graph(model), torch.cuda.graph(g):
        if steps:
            with traceml.trace_step(model):
                torch.nn.functional.cross_entropy(model(x), y).backward()
                opt.step()
        else:
            torch.nn.functional.cross_entropy(model(x), y).backward()
            opt.step()
    return g, opt


def host_loop_us(body, n: int) -> dict:
    """Host time per iteration up to the end of the loop, and up to the synchronise after it."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        body()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return {"loop_us": (t1 - t0) * 1e6 / n, "to_sync_us": (t2 - t0) * 1e6 / n}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mlp-replays", type=int, default=2000)
    ap.add_argument("--resnet-replays", type=int, default=60)
    ap.add_argument("--host-iters", type=int, default=2000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_steps.py measures on the GPU: no CUDA device")
    import traceml_b200 as traceml
    from bench import resnet18
    from traceml_b200 import runtime

    torch.cuda.set_device(0)
    traceml.init(mode="auto")
    torch.manual_seed(0)
    out = {"gpu": gpu_info(0), "device": [], "host": {}}
    eng = runtime.get_engine()
    work = {"micro_mlp": (torch.nn.Linear(8, 8).cuda(), torch.randn(16, 8, device="cuda"),
                          torch.randint(0, 8, (16,), device="cuda"), a.mlp_replays),
            "resnet18_b64": (resnet18().cuda(), torch.randn(64, 3, 224, 224, device="cuda"),
                             torch.randint(0, 10, (64,), device="cuda"), a.resnet_replays)}
    graphs = {name: {"stamps": capture(copy.deepcopy(m), x, y, False)} for name, (m, x, y, _) in work.items()}

    # host time of today's path: trace_step around the replay of the stamps-only graph
    mlp = work["micro_mlp"][0]
    g_st = graphs["micro_mlp"]["stamps"][0]

    def stepped():
        with traceml.trace_step(mlp):
            g_st.replay()

    host_loop_us(stepped, max(10, a.host_iters // 4))
    around = [host_loop_us(stepped, a.host_iters) for _ in range(a.rounds)]
    n_around = eng.step_count

    for name, (m, x, y, _) in work.items():  # from here on the engine is in device-committed mode
        graphs[name]["steps"] = capture(copy.deepcopy(m), x, y, True)
    g_cs = graphs["micro_mlp"]["steps"][0]
    host_loop_us(g_cs.replay, max(10, a.host_iters // 4))
    replays = [host_loop_us(g_cs.replay, a.host_iters) for _ in range(a.rounds)]
    out["host"] = {"workload": "micro_mlp", "iters_per_round": a.host_iters, "rounds": a.rounds,
                   "trace_step_around_replay": {k: spread([r[k] for r in around]) for k in around[0]},
                   "replay_of_captured_step": {k: spread([r[k] for r in replays]) for k in replays[0]},
                   "records": {"around": n_around, "total": eng.step_count}}

    for name, (_, _, _, n) in work.items():
        gs = {arm: graphs[name][arm][0] for arm in ("stamps", "steps")}
        for g in gs.values():
            per_replay_us(g, max(10, n // 4))  # warm-up
        res = {"stamps": [], "steps": []}
        for r in range(a.rounds):
            for arm in (("stamps", "steps") if r % 2 == 0 else ("steps", "stamps")):
                res[arm].append(per_replay_us(gs[arm], n))
        diff = [s - p for s, p in zip(res["steps"], res["stamps"])]
        out["device"].append({"workload": name, "replays_per_round": n, "rounds": a.rounds,
                              "stamps_only_us": spread(res["stamps"]), "captured_step_us": spread(res["steps"]),
                              "added_us": spread(diff),
                              "added_pct": 100.0 * statistics.median(diff) / statistics.median(res["stamps"]),
                              "per_round": res})
    torch.cuda.synchronize()
    out["records_committed"] = eng.step_count
    print(json.dumps(out))


if __name__ == "__main__":
    main()
