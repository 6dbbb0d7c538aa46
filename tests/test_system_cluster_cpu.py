"""CPU: the System section over several nodes.  The oracle against the reference goldens, the
cluster rule engine (tml_diag_system_cluster) and ``build_system_cluster`` against the golden
sections, K6m's shared fold (csrc/tml_sys_sum.h, run here by tml_sys_host_cluster) against
CPython's sum() over the concatenated rows, and the gather orchestration of ``SummaryEngine``
under gloo with one process per node."""
import ctypes as C
import glob
import json
import math
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import system_cases as sc  # noqa: E402
import system_cluster_cases as scc  # noqa: E402
from oracle import system_cluster_oracle, system_oracle  # noqa: E402

GOLDENS = [json.load(open(p)) for p in sorted(glob.glob(os.path.join(HERE, "golden", "system_cluster", "*.json")))
           if not p.endswith("INDEX.json")]
IDS = [g["case"] for g in GOLDENS]


def _drop_gpu_idx(section):
    out = json.loads(json.dumps(section))
    for n in out["nodes"].values():
        n["per_gpu"] = {str(i): {k: v for k, v in q.items() if k != "gpu_idx"} for i, q in n["per_gpu"].items()}
    return out


def _rows(name):
    window, raws, idents = scc.make_case(name)
    return window, [[sc.wire_row(s) for s in raw] for raw in raws], idents


def _node_agg(node):
    return sc.sys_agg_from_oracle({"aggregate": node["aggregate"], "nodes": {"n": node}})


def _cluster_agg(sec):
    from traceml_b200 import _abi

    if not sec["aggregate"]["system_samples"]:
        return _abi.SysAgg()
    return sc.sys_agg_from_oracle({"aggregate": sec["aggregate"], "nodes": {"c": {"per_gpu": {}}}})


def _records_from_oracle(sec, idents):
    """The gathered records and K6m's result as the oracle says they are (every source's record in
    slot order; nodes without samples are records with valid = 0)."""
    from traceml_b200 import _abi, sections

    recs = (_abi.SysNodeRecord * len(idents))()
    keyed = []
    for k, ident in enumerate(idents):
        recs[k].ident = sections.node_ident(ident)
        label = sections.system_node_label(ident)
        if label in sec["nodes"]:
            recs[k].valid = 1
            recs[k].agg = _node_agg(sec["nodes"][label])
            keyed.append((int(label), ident["global_rank"], k))
    out = _abi.SysClusterOut()
    out.agg = _cluster_agg(sec)
    out.n_nodes = len(keyed)
    for j, (_, _, k) in enumerate(sorted(keyed)):
        out.order[j] = k
    return list(recs), out


def test_cluster_structs_mirror_the_c_layouts():
    from traceml_b200 import _abi

    lib = _abi.lib()
    for name, cls in {"tml_sys_part": _abi.SysPart, "tml_sys_node_ident": _abi.SysNodeIdent,
                      "tml_sys_node_record": _abi.SysNodeRecord, "tml_sys_cluster_out": _abi.SysClusterOut}.items():
        assert int(lib.tml_struct_size(name.encode())) == C.sizeof(cls), name
    assert C.sizeof(_abi.SysNodeRecord) % 8 == 0  # K6m's result slot after n records stays 8-B aligned


def test_goldens_cover_the_cluster_geometries():
    assert len(GOLDENS) == 9
    by = {g["case"]: g for g in GOLDENS}
    assert by["partial_coverage_3_of_4"]["section"]["expected_nodes"] == 4
    assert len(by["partial_coverage_3_of_4"]["section"]["nodes"]) == 3
    assert list(by["eleven_nodes"]["section"]["nodes"])[:3] == ["0", "1", "10"]  # string order
    p = by["four_nodes_high_gpu_memory"]["section"]["diagnosis"]["primary"]
    assert p["kind"] == "VERY_HIGH_GPU_MEMORY" and p["scope"]["level"] == "gpu" and p["scope"]["node"] == "2"
    tie = by["tie_broken_by_label"]["section"]["diagnosis"]
    assert [i["evidence"]["scope"]["node"] for i in tie["issues"]] == ["10", "2"]
    assert tie["issues"][0]["score"] == tie["issues"][1]["score"]
    mixed = by["mixed_world_candidates"]
    assert len({math.ceil(i["world_size"] / i["local_world_size"]) for i in mixed["identities"]}) > 1
    assert any(w < max(g["samples"]) for g in GOLDENS for w in [g["window"]])


@pytest.mark.parametrize("g", GOLDENS, ids=IDS)
def test_oracle_equals_golden(g):
    from golden.make_system_golden import wire_digest

    window, rows, idents = _rows(g["case"])
    assert [wire_digest(r) for r in rows] == g["input_sha256"]
    assert idents == g["identities"] and window == g["window"]
    mine = system_cluster_oracle.cluster_section(rows, idents, window)
    assert _drop_gpu_idx(mine) == json.loads(json.dumps(g["section"]))


@pytest.mark.parametrize("g", GOLDENS, ids=IDS)
def test_cluster_rules_and_section_equal_golden(g):
    from traceml_b200 import sections

    window, rows, idents = _rows(g["case"])
    sec = system_cluster_oracle.cluster_section(rows, idents, window)
    recs, out = _records_from_oracle(sec, idents)
    got = sections.build_system_cluster(recs, out)
    want = json.loads(json.dumps(g["section"]))
    assert got["diagnosis"] == want["diagnosis"]
    assert _drop_gpu_idx(got) == want


def test_one_node_cluster_rules_equal_the_node_rules():
    """tml_diag_system_cluster over one node is tml_diag_system: the per-node rule code is shared."""
    from traceml_b200 import sections

    sg = json.load(open(os.path.join(HERE, "golden", "system", "several_issues_g8.json")))
    rows = [sc.wire_row(s) for s in sc.make_raw(sg["case"])]
    sec = system_cluster_oracle.cluster_section([rows], [sg["identity"]], sg["window"])
    recs, out = _records_from_oracle(sec, [sg["identity"]])
    got = sections.build_system_cluster(recs, out)
    assert _drop_gpu_idx(got) == json.loads(json.dumps(sg["section"]))


# ----------------------------------------------------------------------------- K6m's fold
def _host_sum2(x, nblk):
    from traceml_b200 import _abi

    a = np.ascontiguousarray(x, dtype=np.float64)
    out = (C.c_double * 2)()
    _abi.check(_abi.lib().tml_sys_host_sum(a.ctypes.data if len(a) else None, len(a), 2, nblk, out),
               "tml_sys_host_sum")
    return out[0], out[1]


def _host_cluster(recs):
    from traceml_b200 import _abi

    arr = (_abi.SysNodeRecord * len(recs))(*recs)
    out = _abi.SysClusterOut()
    _abi.check(_abi.lib().tml_sys_host_cluster(arr, len(recs), C.byref(out)), "tml_sys_host_cluster")
    return out


def _fold_nodes(parts, node_ranks, nblk=3):
    """One record per node with the K6s fold of its values in cpu_hi / cpu_lo; K6m's result."""
    from traceml_b200 import _abi

    recs = []
    for x, nr in zip(parts, node_ranks):
        r = _abi.SysNodeRecord()
        r.valid = 1
        r.ident.node_rank, r.ident.global_rank = nr, nr * 8
        r.part.cpu_hi, r.part.cpu_lo = _host_sum2(x, nblk)
        r.part.n = len(x)
        r.part.cpu_max = max(x)
        r.part.ts_min, r.part.ts_max = 0.0, 1.0
        recs.append(r)
    return _host_cluster(recs)


def _cluster_families():
    rng = np.random.default_rng(20261017)
    yield "one_decimal_2", [[round(float(v), 1) for v in rng.uniform(0, 100, n)] for n in (10_000, 7)]
    yield "one_decimal_64", [[round(float(v), 1) for v in rng.uniform(0, 100, int(n))]
                             for n in rng.integers(1, 2_000, 64)]
    yield "binades_16", [(rng.uniform(0, 1, int(n)) * 2.0 ** rng.integers(-30, 30, int(n))).tolist()
                         for n in rng.integers(1, 5_000, 16)]
    yield "ties_3", [[1.0], [2.0 ** -53] * 10_001, [3.0 * 2.0 ** -53]]
    yield "ties_half_5", [[2.0 ** 53, 1.0], [1.0, -0.0], [1.0] * 3, [2.0 ** 53], [1.0]]
    yield "watts_2x1e5", [[int(v) / 1000.0 for v in rng.integers(50_000, 700_001, 100_000)] for _ in range(2)]
    yield "uniform_8", [rng.uniform(0, 100, int(n)).tolist() for n in rng.integers(1, 20_000, 8)]
    yield "single_samples_64", [[float(v)] for v in rng.uniform(0, 100, 64)]


@pytest.mark.parametrize("name,parts", list(_cluster_families()), ids=[n for n, _ in _cluster_families()])
def test_cluster_fold_equals_sum_over_the_concatenated_rows(name, parts):
    """The nodes arrive in a shuffled slot order; K6m folds them by node rank, the reference's
    row order, and the rounded mean is CPython's sum() / len() over the concatenated rows."""
    rng = np.random.default_rng(len(parts))
    node_ranks = rng.permutation(len(parts)).tolist()
    out = _fold_nodes(parts, node_ranks)
    concat = [v for nr in range(len(parts)) for v in parts[node_ranks.index(nr)]]
    assert out.n_nodes == len(parts) and out.n_dup == 0
    assert out.agg.n == len(concat)
    assert out.agg.cpu_avg == sum(concat) / len(concat)
    assert out.agg.cpu_peak == max(concat)
    assert [node_ranks[out.order[j]] for j in range(len(parts))] == list(range(len(parts)))


def test_one_node_fold_is_the_node_finish_bit_for_bit():
    """K = 1: folding one part and rounding gives the node's own K6s result."""
    x = np.random.default_rng(3).uniform(0, 100, 12_345).tolist()
    hi, lo = _host_sum2(x, 7)
    out = _fold_nodes([x], [0], nblk=7)
    assert out.agg.cpu_avg == (hi + lo) / len(x)


def test_duplicate_labels_keep_the_lowest_global_rank():
    from traceml_b200 import _abi

    recs = []
    for gr, nr, n in ((24, 1, 5), (8, 1, 7), (0, 0, 3), (16, -1, 2), (40, 5, 0)):
        r = _abi.SysNodeRecord()
        r.valid = 1 if n else 0
        r.ident.global_rank, r.ident.node_rank = gr, nr
        r.part.n, r.part.cpu_hi = n, float(n)
        r.part.ts_min, r.part.ts_max = 0.0, 0.0
        recs.append(r)
    out = _host_cluster(recs)
    # labels: "1" twice (global ranks 24 and 8 -> 8 kept), "0", "16" (no node rank); "5" is empty
    assert (out.n_nodes, out.n_dup) == (3, 1)
    assert list(out.order[:3]) == [2, 1, 3] and out.order[3] == -1
    assert out.agg.n == 3 + 7 + 2


def test_no_valid_record_is_no_data():
    from traceml_b200 import _abi, sections

    r = _abi.SysNodeRecord()
    r.ident = sections.node_ident({"global_rank": 0, "node_rank": 0})
    out = _host_cluster([r])
    assert out.n_nodes == 0 and out.agg.n == 0
    sec = sections.build_system_cluster([r], out)
    assert sec["nodes"] == {} and sec["expected_nodes"] == 1
    assert sec["diagnosis"]["primary"]["kind"] == "NO_DATA"


# ----------------------------------------------------------------------------- gloo: one process per node
def _pack_numpy(raw, identity, max_rows):
    """A node record from the node's raw samples, computed in numpy (the K6s stand-in): the
    oracle's node aggregates and the unrounded part the fold needs."""
    from traceml_b200 import _abi, sections

    rec = _abi.SysNodeRecord()
    rec.ident = sections.node_ident(identity)
    win = raw[-max_rows:]
    if not win:
        return rec
    rows = [sc.wire_row(s) for s in win]
    sec = system_oracle.system_section(rows, identity, max_rows)
    rec.valid = 1
    rec.agg = _node_agg(next(iter(sec["nodes"].values())))
    d = [system_oracle.derived_row(r) for r in rows]
    p = rec.part
    p.cpu_hi, p.cpu_lo = _host_sum2([x["cpu"] for x in d], 1)
    p.cpu_max = max(x["cpu"] for x in d)
    p.ts_min, p.ts_max = min(x["ts"] for x in d), max(x["ts"] for x in d)
    with_gpu = [x for x in d if x["util_avg"] is not None]
    for k, col in enumerate(("util", "mem", "temp", "power")):
        vals = [x[col + "_avg"] for x in with_gpu]
        p.d_hi[k], p.d_lo[k] = _host_sum2(vals, 1) if vals else (0.0, 0.0)
        p.d_max[k] = max((x[col + "_peak"] for x in with_gpu), default=-math.inf)
    p.ram_sum = sum(int(s["ram_used"]) for s in win)
    p.ram_max = max(int(s["ram_used"]) for s in win)
    p.ram_total_max = max(int(s["ram_total"]) for s in win)
    p.n, p.n_gpu = len(win), len(with_gpu)
    p.avail = int(any(s["gpu_available"] for s in win))
    p.gpu_count = max(int(s["gpu_count"]) for s in win)
    p.n_gpus = max(len(s["gpus"]) for s in win)
    return rec


def _cluster_worker(rank, world, case, one_node, init_file, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ.update({"WORLD_SIZE": str(world), "RANK": str(rank)})
    if one_node:
        os.environ.update({"LOCAL_WORLD_SIZE": str(world), "LOCAL_RANK": str(rank), "GROUP_RANK": "0"})
    else:
        os.environ.update({"LOCAL_WORLD_SIZE": "1", "LOCAL_RANK": "0", "GROUP_RANK": str(rank)})
    import torch
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world)
    from fake_engine import FakeEngine
    import replay
    from traceml_b200 import _abi, sections
    from traceml_b200.reduce import TorchDistComm

    class SystemFakeEngine(FakeEngine):
        """The engine double with a system ring: K6s, the record pack and K6m in numpy (the fold
        itself is the shared native one, tml_sys_host_cluster)."""

        def __init__(self, recs, procs, raw, identity):
            super().__init__(recs, procs)
            self.raw, self.identity, self.rows_n = raw, identity, None

        @property
        def sys_count(self):
            return len(self.raw)

        def sys_reduce_beside(self, max_rows, stream=0):
            self.rows_n = int(max_rows)

        def sys_reduce_collect(self):
            sec = system_oracle.system_section([sc.wire_row(s) for s in self.raw], self.identity, self.rows_n)
            return sc.sys_agg_from_oracle(sec)

        def sys_node_pack(self, ident, d_record, stream=0):
            rec = _pack_numpy(self.raw, self.identity, self.rows_n) if ident is not None else _abi.SysNodeRecord()
            if ident is not None:
                assert bytes(ident) == bytes(sections.node_ident(self.identity))
            else:
                rec.ident.node_rank = -1
            d_record.numpy()[:] = np.frombuffer(bytes(rec), dtype=np.uint8)

        def sys_cluster_launch(self, d_records, n, stream=0):
            size = C.sizeof(_abi.SysNodeRecord)
            buf = d_records.numpy()
            recs = (_abi.SysNodeRecord * n).from_buffer_copy(buf[: n * size].tobytes())
            out = _abi.SysClusterOut()
            _abi.check(_abi.lib().tml_sys_host_cluster(recs, n, C.byref(out)), "tml_sys_host_cluster")
            buf[n * size: n * size + C.sizeof(out)] = np.frombuffer(bytes(out), dtype=np.uint8)
            self.last = buf.copy()

        def sys_cluster_collect(self, n):
            size = C.sizeof(_abi.SysNodeRecord)
            recs = list((_abi.SysNodeRecord * n).from_buffer_copy(self.last[: n * size].tobytes()))
            return recs, _abi.SysClusterOut.from_buffer_copy(self.last[n * size:].tobytes())

    window, raws, idents = scc.make_case(case)
    recs = replay.make_step_replay("balanced", world, 120, seed=3)
    procs = replay.make_proc_replay("normal", world, 50, seed=3)
    from traceml_b200.reporting import default_identity

    ident = default_identity(rank, world)
    raw = raws[rank]
    if not one_node:  # the case's node streams; identities as the launcher's environment gives them
        idents[rank] = ident
    eng = SystemFakeEngine(recs[rank], procs[rank], raw, ident)
    comm = TorchDistComm()
    gathers = []
    inner = comm.all_gather_into

    def counting(out, inp):
        if inp.dtype == torch.uint8 and inp.numel() == C.sizeof(_abi.SysNodeRecord):
            gathers.append(out.numel())
        inner(out, inp)

    comm.all_gather_into = counting
    se = sections.SummaryEngine([eng], comm, exchange="a2a", ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1)
    se.reducer.device = torch.device("cpu")
    res = se.build(window, window)
    torch.save({"system": res["system"], "gathers": gathers, "multi_node": se.multi_node, "ident": ident},
               os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.parametrize("case,one_node", [("two_nodes_g8", False), ("cpu_only_node", False),
                                           ("two_nodes_g8", True)])
def test_gloo_world2_gathers_one_record_per_node(case, one_node):
    import torch
    import torch.multiprocessing as mp

    world = 2
    with tempfile.TemporaryDirectory() as td:
        mp.spawn(_cluster_worker, args=(world, case, one_node, os.path.join(td, "init"), td), nprocs=world, join=True)
        got = [torch.load(os.path.join(td, f"r{r}.pt"), weights_only=False) for r in range(world)]
    window, raws, _ = scc.make_case(case)
    rows = [[sc.wire_row(s) for s in raw] for raw in raws]
    if one_node:  # today's path: comm index 0 is the one source, no record crosses the group
        assert [g["multi_node"] for g in got] == [False, False]
        assert [g["gathers"] for g in got] == [[], []]
        return
    assert [g["multi_node"] for g in got] == [True, True]
    assert all(len(g["gathers"]) == 1 for g in got)  # one record gather per build, on every rank
    assert [g["ident"]["node_rank"] for g in got] == [0, 1]
    assert [g["ident"]["local_rank"] for g in got] == [0, 0]
    assert got[1]["system"] is None
    want = system_cluster_oracle.cluster_section(rows, [g["ident"] for g in got], window)
    assert _drop_gpu_idx(got[0]["system"]) == _drop_gpu_idx(want)
