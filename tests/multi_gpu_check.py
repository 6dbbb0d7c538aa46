"""Multi-GPU parity check, launched by torchrun (one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29533 tests/multi_gpu_check.py

Every rank loads ITS replay records, the job runs the cross-rank reduce with the
fused NVLink peer-load exchange ("p2p"), the NCCL all-gather ("nccl") and the
step-sharded NCCL all-to-all ("a2a"); rank 0 checks them against each other and
the oracle (test infrastructure).  Then the live tick (StepCombined twin) runs
across the real ranks and is checked against its oracle."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from helpers import assert_struct, oracle_mem_rows, oracle_proc_rows, oracle_time_rows, plain, strip_device
    from oracle import process_oracle, step_memory_oracle, step_time_oracle
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine
    from traceml_b200.reduce import TorchDistComm

    failures = 0
    for scenario, S, W in (("straggler", 700, 10_000), ("ragged", 900, 256), ("empty_rank", 300, 10_000),
                           ("no_overlap", 120, 10_000), ("duplicates", 400, 100), ("lagging", 700, 3),
                           ("input_straggler", 200_000, 150_000)):
        gen = "duplicates" if scenario == "lagging" else scenario
        recs_all = replay.make_step_replay(gen, world, S, seed=11) if S <= 1000 else None
        if scenario == "lagging":  # the last rank is far behind: the memory candidate limit (20 W) binds
            recs_all[world - 1] = recs_all[world - 1][:150]
        mine = (recs_all[rank] if recs_all is not None else
                replay.make_step_replay(scenario, world, S, seed=11, only_ranks=[rank])[rank])
        procs = replay.make_proc_replay("overhang", world, 500, seed=11, only_ranks=[rank])[rank]
        results = {}
        # (label, exchange, native sequencing): the C++ driver (tml_reduce_run, NCCL on torch's
        # communicator) and the Python driver must agree bit for bit
        for label, mode, native in (("p2p", "p2p", True), ("nccl", "nccl", False), ("a2a", "a2a", True),
                                    ("p2p_py", "p2p", False), ("a2a_py", "a2a", False), ("auto", "auto", True)):
            eng = Engine(device=local, rank=rank, world=world, ring_slots=max(64, len(mine) + 8), proc_slots=1024)
            if len(mine):
                eng.load_steps(mine)
            eng.load_procs(procs)
            torch.cuda.synchronize()
            se = sections.SummaryEngine([eng], TorchDistComm(), exchange=mode, native=native,
                                        ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=world)
            assert se.reducer._native_ok() == native, (label, se.reducer._native_ok())
            res = se.build(W, W)
            import time as _t
            torch.cuda.synchronize(); dist.barrier(); t0 = _t.perf_counter()
            res = se.build(W, W)
            torch.cuda.synchronize(); res["_ms"] = (_t.perf_counter() - t0) * 1e3
            if mode != "auto":
                assert res["reduce"].exchange == mode, (label, res["reduce"].exchange)
            results[label] = res
            dist.barrier()
            eng.close()
        if rank == 0:
            try:
                a, b = results["p2p"], results["nccl"]
                assert_struct(plain(a["step_time"]), plain(b["step_time"]), f"{scenario}: p2p == nccl", rel=0.0)
                c = results["a2a"]
                for other in ("a2a", "p2p_py", "a2a_py", "auto"):
                    o_ = results[other]
                    assert_struct(plain(a["step_time"]), plain(o_["step_time"]), f"{scenario}: p2p == {other}", rel=0.0)
                    assert_struct(plain(a["step_memory"]), plain(o_["step_memory"]), f"mem p2p == {other}", rel=0.0)
                    assert_struct(plain(a["process"]), plain(o_["process"]), f"proc p2p == {other}", rel=0.0)
                assert_struct(plain(a["step_memory"]["diagnosis"]), plain(b["step_memory"]["diagnosis"]), "mem p2p == nccl", rel=0.0)
                if recs_all is not None:
                    ref = step_time_oracle.step_time_section(oracle_time_rows(recs_all, W), max_rows=W)
                    g = a["step_time"]
                    assert_struct(plain(g["data"]), plain({k: ref["data"][k] for k in g["data"]}), "data")
                    assert_struct(plain(g["diagnosis"]), plain(ref["diagnosis"]), "diagnosis")
                    mref = step_memory_oracle.step_memory_section(
                        oracle_mem_rows(recs_all), window_size=W, gpu_total_bytes=a["step_memory"]["gpu_total_bytes"])
                    assert_struct(strip_device(plain(a["step_memory"]["diagnosis"]))["primary"],
                                  strip_device(plain(mref["diagnosis"]))["primary"], "mem.primary")
                    procs_all = replay.make_proc_replay("overhang", world, 500, seed=11)
                    pref = process_oracle.process_section(oracle_proc_rows(procs_all, world), max_rows=W)
                    assert_struct(plain(a["process"]["primary"]), plain(pref["diagnosis"]["primary"]), "proc.primary")
                else:
                    # large window: the numpy oracle (pinned == row-level oracle == reference); the
                    # per-rank sums must be BIT-exact (K3e, deferred beside K4 in the native driver)
                    from oracle import fast_oracle

                    big = replay.make_step_replay(scenario, world, S, seed=11)
                    fref = fast_oracle.step_time_section(big, max_rows=W)
                    g = a["step_time"]
                    assert plain(g["data"]["aligned_summary"]) == plain(fref["data"]["aligned_summary"]), "aligned sums"
                    assert plain(g["data"]["per_global_rank_summary"]) == plain(fref["data"]["per_global_rank_summary"])
                    assert_struct(plain(g["diagnosis"]), plain(fref["diagnosis"]), "big.diagnosis")
                    assert_struct(plain(g["global"]), plain(fref["global"]), "big.global")
                    mref = fast_oracle.step_memory_section(big, window_size=W,
                                                           gpu_total_bytes=a["step_memory"]["gpu_total_bytes"])
                    assert plain(a["step_memory"]["per_global_rank"]) == plain(mref["per_global_rank"])
                    assert_struct(plain(a["step_memory"]["global"]), plain(mref["global"]), "big.mem.global")
                    assert a["step_time"]["diagnosis"]["primary"]["kind"] == "INPUT_STRAGGLER"
                    assert a["step_time"]["data"]["aligned_window"]["steps_analyzed"] == W
                print(f"[multi_gpu_check] {scenario} R={world} W={W}: OK "
                      f"({a['step_time']['diagnosis']['primary']['status'] if a['step_time']['diagnosis'] else None}); "
                      + ", ".join(f"{k} {v['_ms']:.3f} ms" for k, v in results.items())
                      + f" (auto -> {results['auto']['reduce'].exchange})")
            except AssertionError as exc:
                failures += 1
                print(f"[multi_gpu_check] {scenario}: FAILED {exc}")
    # ---- process aggregates whose byte totals pass 2^53 on every rank (10^4 samples of ~1.8 TiB):
    # the exact u64 sums must cross every exchange intact, native (pack_proc) and Python drivers
    import process_cases as pc

    P = 10_000
    steps = replay.make_step_replay("straggler", world, 300, seed=5)[rank]
    pres = {}
    for label, mode, native in (("nccl", "nccl", False), ("a2a", "a2a", True), ("a2a_py", "a2a", False),
                                ("auto", "auto", True)):
        eng = Engine(device=local, rank=rank, world=world, ring_slots=512, proc_slots=P + 8)
        eng.load_steps(steps)
        eng.load_procs(pc.make("bytes_1t8", P, seed=12, rank=rank))
        torch.cuda.synchronize()
        se = sections.SummaryEngine([eng], TorchDistComm(), exchange=mode, native=native,
                                    ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=world)
        pres[label] = plain(se.build(256, P)["process"])
        dist.barrier()
        eng.close()
    if rank == 0:
        try:
            procs_all = {r: pc.make("bytes_1t8", P, seed=12, rank=r) for r in range(world)}
            pref = process_oracle.process_section(oracle_proc_rows(procs_all, world), max_rows=P)
            for label, got in pres.items():
                assert got["aggregate"] == plain(pref["data"]["aggregate"]), f"proc > 2^53 {label}: aggregate"
                assert got["per_global_rank"] == plain(pref["data"]["per_global_rank"]), f"proc > 2^53 {label}"
                assert got["primary"] == plain(pref["diagnosis"]["primary"]), f"proc > 2^53 {label}: primary"
            print(f"[multi_gpu_check] process bytes > 2^53 R={world}: OK ({', '.join(pres)})")
        except AssertionError as exc:
            failures += 1
            print(f"[multi_gpu_check] process bytes > 2^53: FAILED {exc}")

    # ---- live tick across the real ranks
    from oracle import live_oracle
    from traceml_b200 import records as rec_mod
    from traceml_b200.live import StepCombinedComputer, StepMemoryCombinedComputer

    for scenario, S, W in (("ragged", 700, 100), ("input_straggler", 460, 100), ("duplicates", 300, 64)):
        recs_all = replay.make_step_replay(scenario, world, S, seed=13)
        eng = Engine(device=local, rank=rank, world=world, ring_slots=max(64, len(recs_all[rank]) + 16),
                     proc_slots=64)
        if len(recs_all[rank]):
            eng.load_steps(recs_all[rank])
        torch.cuda.synchronize()
        comp = StepCombinedComputer([eng], TorchDistComm(), window_size=W)
        import time as _t
        got = comp.compute_cli()
        t0 = _t.perf_counter()
        for _ in range(5):
            got = comp.compute_cli()
        tick_ms = (_t.perf_counter() - t0) / 5 * 1e3
        dash = comp.compute_dashboard()
        mem = StepMemoryCombinedComputer([eng], TorchDistComm(), window_size=W).compute()
        dist.barrier()
        eng.close()
        if rank == 0:
            try:
                rows = {r: [rec_mod.step_record_to_wire(x, device=f"cuda:{r}") for x in recs_all[r]]
                        for r in recs_all}
                assert_struct(plain(got), plain(live_oracle.live_step_time(rows, window=W)), "live.cli", rel=1e-9)
                assert_struct(plain(dash), plain(live_oracle.live_step_time(
                    rows, window=W, include_series=False, include_rank_heatmap=True)), "live.dash", rel=1e-9)
                mrows = {r: [(int(s_), float(a_), float(v_)) for s_, a_, v_ in
                             zip(recs_all[r]["step"], recs_all[r]["peak_alloc"], recs_all[r]["peak_resv"])]
                         for r in recs_all}
                for m in mem["metrics"]:
                    m.pop("device", None)
                assert_struct(plain(mem), plain(live_oracle.live_step_memory(mrows, window=W, gpu_available=True)),
                              "live.mem", rel=1e-9)
                print(f"[multi_gpu_check] live {scenario} R={world} W={W}: OK ({got['status_message']}); "
                      f"tick {tick_ms:.3f} ms")
            except AssertionError as exc:
                failures += 1
                print(f"[multi_gpu_check] live {scenario}: FAILED {exc}")
    t = torch.tensor([failures], device="cuda")
    dist.broadcast(t, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(t.item()) else 0)


if __name__ == "__main__":
    main()
