"""Multi-node System section check on one host, launched by torchrun (one rank per GPU, 2 GPUs):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29534 tests/multi_node_system_check.py

Each rank plays a node of its own: it sets LOCAL_RANK=0, LOCAL_WORLD_SIZE=1 and GROUP_RANK=<rank>
before anything reads them, so every rank is its node's System source.  Each loads a seeded node
stream into its engine's system ring and calls final_summary(); rank 0's System section (and,
where the reference is installed, its System payload) must equal the oracle's cluster section
over the same streams.  With fewer than two GPUs it says so and exits without running."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def _drop_gpu_idx(section):
    out = json.loads(json.dumps(section))
    for n in out["nodes"].values():
        n["per_gpu"] = {str(i): {k: v for k, v in q.items() if k != "gpu_idx"} for i, q in n["per_gpu"].items()}
    return out


def main():
    if torch.cuda.device_count() < 2:
        print("multi_node_system_check: fewer than two GPUs; not run")
        return 0
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    os.environ.update({"LOCAL_RANK": "0", "LOCAL_WORLD_SIZE": "1", "GROUP_RANK": str(rank)})
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import system_cases as sc
    from oracle import system_cluster_oracle
    from traceml_b200 import reporting, runtime, sections
    from traceml_b200.reduce import TorchDistComm
    from traceml_b200.summary import final_summary

    W = 10_000
    raws = [sc.make_raw("normal_g8" if k % 2 == 0 else "very_high_gpu_memory_g8", seed=k) for k in range(world)]
    idents = [reporting.default_identity(k, world) for k in range(world)]
    for k, i in enumerate(idents):  # what each rank's environment says about itself
        i.update({"local_rank": 0, "local_world_size": 1, "node_rank": k})
    eng = runtime.get_engine()
    eng.load_sys(sc.sys_records(raws[rank]))
    torch.cuda.synchronize()
    want = system_cluster_oracle.cluster_section([[sc.wire_row(s) for s in r] for r in raws], idents, W)

    failures = 0
    se = sections.SummaryEngine([eng], TorchDistComm())
    got = se.build(W, W)["system"]
    if rank == 0:
        if not se.multi_node or _drop_gpu_idx(got) != _drop_gpu_idx(want):
            print("FAIL: SummaryEngine System section differs from the oracle", file=sys.stderr)
            failures += 1
    out = final_summary(window_rows=W)
    if rank == 0:
        if out is None:
            print("FAIL: final_summary returned None", file=sys.stderr)
            failures += 1
        elif reporting.reference_available():
            from traceml.reporting.sections.system.builder import build_system_payload

            from golden.make_system_golden import _plain

            ref = _plain(build_system_payload(*reporting.to_reference_system(want)))
            if json.loads(json.dumps(out["system"], default=str)) != json.loads(json.dumps(ref, default=str)):
                print("FAIL: final_summary System payload differs from the oracle's", file=sys.stderr)
                failures += 1
        print(f"multi_node_system_check: {world} nodes, {'FAIL' if failures else 'ok'}")
    t = torch.tensor([failures], device="cuda")
    dist.all_reduce(t)
    dist.destroy_process_group()
    return int(t.item() > 0)


if __name__ == "__main__":
    sys.exit(main())
