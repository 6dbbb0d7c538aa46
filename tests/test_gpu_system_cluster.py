"""GPU: the System section over several nodes, on one device.

K simulated nodes: K engines, each loaded with one node's samples by tml_sys_load, each runs K6s
and packs its node record into consecutive slots of one device buffer -- what the all-gather of a
multi-node run leaves on comm index 0.  Then K6m (k_sys_cluster), the cluster rules and
``build_system_cluster``:
- for every cluster golden the section equals the oracle's and the golden's (data and diagnosis,
  ``==`` on floats), and the kept builder's payload and text equal the golden's;
- K = 1, 2, 11, 64 nodes, rings that wrapped, windows below and above the retained count: the
  section equals ``system_cluster_oracle.cluster_section`` with ``==``;
- each record carries its node's K6s result bit for bit;
- a single-node build still runs exactly one System launch (K6s), no pack and no K6m, and its
  section is the one-node section of the oracle.
"""
import ctypes as C
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import system_cases as sc  # noqa: E402
import system_cluster_cases as scc  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN_DIR = os.path.join(HERE, "golden", "system_cluster")
GOLDENS = [json.load(open(os.path.join(GOLDEN_DIR, f))) for f in sorted(os.listdir(GOLDEN_DIR))
           if f.endswith(".json") and f != "INDEX.json"]


@pytest.fixture(scope="module")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _drop_gpu_idx(section):
    out = json.loads(json.dumps(section))
    for n in out["nodes"].values():
        n["per_gpu"] = {str(i): {k: v for k, v in q.items() if k != "gpu_idx"} for i, q in n["per_gpu"].items()}
    return out


def _cluster_on_gpu(raws, idents, window, slots=1024):
    """K engines -> K6s each -> records packed into one buffer -> K6m on the first engine."""
    import torch

    from traceml_b200 import _abi, sections
    from traceml_b200.engine import Engine

    K = len(raws)
    rec = C.sizeof(_abi.SysNodeRecord)
    buf = torch.full((K * rec + C.sizeof(_abi.SysClusterOut),), 0xAB, dtype=torch.uint8, device="cuda")
    stream = int(torch.cuda.current_stream().cuda_stream)
    engines = [Engine(device=0, rank=k, world=K, ring_slots=64, proc_slots=slots) for k in range(K)]
    try:
        node_aggs = []
        for k, (raw, eng) in enumerate(zip(raws, engines)):
            if raw:
                eng.load_sys(sc.sys_records(raw))
            eng.sys_reduce_launch(window, stream)
            node_aggs.append(eng.sys_reduce_collect())
            l0 = eng.launch_count
            eng.sys_node_pack(sections.node_ident(idents[k]), buf[k * rec:], stream)
            assert eng.launch_count - l0 == 1
        l0 = engines[0].launch_count
        engines[0].sys_cluster_launch(buf, K, stream)
        records, out = engines[0].sys_cluster_collect(K)
        assert engines[0].launch_count - l0 == 1
    finally:
        for e in engines:
            e.close()
    for k, r in enumerate(records):
        assert r.valid == (1 if node_aggs[k].n else 0)
        assert bytes(r.ident) == bytes(sections.node_ident(idents[k]))
        if r.valid:
            assert bytes(r.agg) == bytes(node_aggs[k])
    return sections.build_system_cluster(records, out), out


@pytest.mark.parametrize("g", GOLDENS, ids=[g["case"] for g in GOLDENS])
def test_cluster_section_equals_golden(cuda, g):
    from oracle import system_cluster_oracle
    from traceml_b200 import reporting

    window, raws, idents = scc.make_case(g["case"])
    got, _ = _cluster_on_gpu(raws, idents, window)
    rows = [[sc.wire_row(s) for s in raw] for raw in raws]
    want = system_cluster_oracle.cluster_section(rows, idents, window)
    assert _drop_gpu_idx(got) == _drop_gpu_idx(want)
    assert _drop_gpu_idx(got) == json.loads(json.dumps(g["section"]))
    if reporting.reference_available():
        from golden.make_system_golden import _plain
        from traceml.reporting.sections.system.builder import build_system_payload
        from traceml.reporting.sections.system.formatter import format_system_section_text

        payload = build_system_payload(*reporting.to_reference_system(got))
        assert json.loads(json.dumps(_plain(payload))) == json.loads(json.dumps(g["payload"]))
        assert format_system_section_text(payload) == g["text"]


@pytest.mark.parametrize("K,slots,window,seed", [
    (1, 1024, 10_000, 1), (2, 1024, 10_000, 2), (2, 100, 10_000, 3),   # 100 slots: rings that wrapped
    (11, 1024, 50, 4),                                                  # window below the retained count
    (11, 160, 10_000, 5), (64, 1024, 10_000, 6), (64, 128, 77, 7),
])
def test_cluster_section_equals_oracle_at_scale(cuda, K, slots, window, seed):
    from oracle import system_cluster_oracle

    raws, idents = scc.random_nodes(K, seed)
    if K > 2:
        raws[K // 2] = []  # a leader without samples
    got, out = _cluster_on_gpu(raws, idents, window, slots)
    keep = [raw[-min(slots, window):] for raw in raws]
    rows = [[sc.wire_row(s) for s in raw] for raw in keep]
    want = system_cluster_oracle.cluster_section(rows, idents, window)
    assert out.n_nodes == sum(1 for r in raws if r) and out.n_dup == 0
    assert _drop_gpu_idx(got) == _drop_gpu_idx(want)


def test_single_node_build_is_unchanged(cuda):
    """One node: the build launches K6s and nothing else for the System section, gathers nothing,
    and its section is the one-node section."""
    import torch

    import replay
    from oracle import system_oracle
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=4096, proc_slots=8192)
    try:
        eng.load_steps(replay.make_step_replay("balanced", 1, 2_000, seed=7)[0])
        eng.load_procs(replay.make_proc_replay("normal", 1, 500, seed=7)[0])
        torch.cuda.synchronize()
        se = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1,
                                    system_identity=sc.IDENTITY)
        assert not se.multi_node
        l0 = eng.launch_count
        se.build(10_000, 10_000)
        launches_empty = eng.launch_count - l0
        raw = sc.make_raw("several_issues_g8")
        eng.load_sys(sc.sys_records(raw))
        torch.cuda.synchronize()
        l0 = eng.launch_count
        res = se.build(10_000, 10_000)
        assert eng.launch_count - l0 == launches_empty + 1
    finally:
        eng.close()
    g = json.load(open(os.path.join(HERE, "golden", "system", "several_issues_g8.json")))
    want = system_oracle.system_section([sc.wire_row(s) for s in raw], sc.IDENTITY, 10_000)
    assert _drop_gpu_idx(res["system"]) == _drop_gpu_idx(want) == json.loads(json.dumps(g["section"]))
