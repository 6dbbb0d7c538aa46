"""The final summary's sections from the device-side reduce.

The GPU-native counterpart of
``src/traceml/reporting/sections/{step_time,step_memory,process,system}/__init__.py``
(``load -> to_diagnosis_input -> diagnose``): ``load`` is the cross-rank window
reduce on the GPUs (``reduce.WindowReducer``), ``diagnose`` is the C++ rule
engine (``csrc/tml_diag.cpp``).  The Step-Time, Step-Memory and Process objects come
from ``tml_sections_json`` (``csrc/tml_sections.cpp``) in one JSON parse, whichever driver
sequenced the reduce; the System section is assembled here.  The objects carry the
reference's field names; ``reporting.py`` turns them into the reference's own dataclasses
for the kept payload builders.
"""

from __future__ import annotations

import math
import os
from typing import Any, Dict, Optional, Sequence

from . import _abi
from .reduce import WindowReducer, _stream_of


# ----------------------------------------------------------------------------- process
def build_process(aggs: Dict[int, Dict[str, Any]]) -> Dict[str, Any]:
    """The Process section straight from ``tml_diag_process``.  aggs[rank] = ProcAgg fields +
    ram_total + gpu_count, which may differ per rank here (``SummaryEngine.build`` passes one
    host's constants for every rank)."""
    din = _abi.ProcDiagIn()
    ranks = sorted(aggs)
    din.n_ranks = len(ranks)
    for i, r in enumerate(ranks):
        a = aggs[r]
        din.ranks[i] = int(r)
        for f, _ in _abi.ProcAgg._fields_:
            setattr(din.agg[i], f, a[f])
        din.ram_total[i] = float(a.get("ram_total", 0.0))
        din.gpu_count[i] = int(a.get("gpu_count", 0))
    return _abi.diag_json("tml_diag_process", din)


def proc_agg_dict(agg: _abi.ProcAgg, *, ram_total: float, gpu_count: int) -> Dict[str, Any]:
    d = {f: getattr(agg, f) for f, _ in _abi.ProcAgg._fields_}
    d["ram_total"] = float(ram_total)
    d["gpu_count"] = int(gpu_count)
    return d


# ----------------------------------------------------------------------------- system
def system_node_label(identity: Dict[str, Any]) -> str:
    """SystemNodeIdentity.label (reporting/sections/system/loader.py:78-81)."""
    if identity.get("node_rank") is not None:
        return str(int(identity["node_rank"]))
    return str(int(identity.get("global_rank") or 0))


def build_system(agg: Optional[_abi.SysAgg], identity: Dict[str, Any]) -> Dict[str, Any]:
    """The System section of the engine's one node from the K6s aggregates: the cluster aggregate,
    ``nodes``, ``expected_nodes`` (loader.py:159-167, 300-359) and the diagnosis of the C++ rule
    engine (``tml_diag_system``).  ``agg`` None or empty: no samples, the reference's NO_DATA."""
    if agg is None:
        agg = _abi.SysAgg()
    label = system_node_label(identity)
    din = _abi.SysDiagIn()
    din.node_rank = int(identity["node_rank"]) if identity.get("node_rank") is not None else -1
    din.node_label = label.encode()[:31]
    din.agg = agg
    d = _abi.diag_json("tml_diag_system", din)
    n = int(agg.n)
    nodes: Dict[str, Any] = {}
    expected = 1
    if n:
        ident = {"label": label}
        ident.update({k: identity.get(k) for k in ("node_rank", "hostname", "global_rank", "local_rank",
                                                   "local_world_size", "world_size")})
        nodes[label] = {"identity": ident, "aggregate": dict(d["aggregate"]),
                        "per_gpu": {int(k): v for k, v in d["per_gpu"].items()}}
        world, lws = identity.get("world_size"), identity.get("local_world_size")
        if world and lws:
            expected = max(1, int(math.ceil(float(world) / float(lws))))
    return {"aggregate": d["aggregate"], "nodes": nodes, "expected_nodes": expected,
            "diagnosis": {"primary": d["primary"], "issues": d["issues"]}}


def multi_node_run(comm) -> bool:
    """Is the System section gathered across nodes?  Only when the run has more than one process
    and, by the launcher's environment, more than one node: ``ceil(WORLD_SIZE / LOCAL_WORLD_SIZE)
    > 1``.  Every rank reads the same two variables, so every rank takes the same branch of what
    is a collective."""
    if int(getattr(comm, "world", 1)) <= 1:
        return False
    try:
        world, lws = int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_WORLD_SIZE"])
    except (KeyError, ValueError):
        return False
    return lws > 0 and math.ceil(world / lws) > 1


def node_ident(identity: Dict[str, Any]) -> _abi.SysNodeIdent:
    """The record identity of a System source (``reporting.default_identity`` fields)."""
    i = _abi.SysNodeIdent()
    i.global_rank = int(identity.get("global_rank") or 0)
    i.local_rank = int(identity.get("local_rank") or 0)
    i.node_rank = int(identity["node_rank"]) if identity.get("node_rank") is not None else -1
    i.world_size = int(identity.get("world_size") or 0)
    i.local_world_size = int(identity.get("local_world_size") or 0)
    i.hostname = str(identity.get("hostname") or "").encode()[: _abi.TML_HOSTNAME_MAX - 1]
    return i


def _record_identity(rec: _abi.SysNodeRecord) -> Dict[str, Any]:
    i = rec.ident
    ident = {"node_rank": int(i.node_rank) if i.node_rank >= 0 else None,
             "hostname": i.hostname.decode("utf-8", "replace"), "global_rank": int(i.global_rank),
             "local_rank": int(i.local_rank), "local_world_size": int(i.local_world_size),
             "world_size": int(i.world_size)}
    return dict({"label": system_node_label(ident)}, **ident)


def build_system_cluster(host_records: Sequence[_abi.SysNodeRecord], cluster: _abi.SysClusterOut) -> Dict[str, Any]:
    """The System section of every node from the gathered records and K6m's result: the same
    shape as ``build_system``, with one entry per node in ``nodes`` (in the string order of their
    labels, loader.py:300-359), the cluster aggregate over all their samples, the reference's
    ``expected_nodes`` (loader.py:159-167) and the cluster-wide diagnosis of
    ``tml_diag_system_cluster``."""
    kept = [host_records[int(k)] for k in cluster.order[: int(cluster.n_nodes)]]
    idents = [_record_identity(r) for r in kept]
    by_label = sorted(zip(idents, kept), key=lambda p: p[0]["label"])
    din = (_abi.SysDiagIn * max(1, len(by_label)))()
    for k, (ident, rec) in enumerate(by_label):
        din[k].node_rank = ident["node_rank"] if ident["node_rank"] is not None else -1
        din[k].node_label = ident["label"].encode()[:31]
        din[k].agg = rec.agg
    d = _abi.diag_system_cluster(din, len(by_label), cluster.agg)
    nodes = {ident["label"]: {"identity": ident, "aggregate": d["nodes"][ident["label"]]["aggregate"],
                              "per_gpu": {int(k): v for k, v in d["nodes"][ident["label"]]["per_gpu"].items()}}
             for ident, _ in by_label}
    cands = {int(math.ceil(float(i["world_size"]) / float(i["local_world_size"])))
             for i in idents if i["world_size"] and i["local_world_size"]}
    expected = max(1, cands.pop()) if len(cands) == 1 else max(1, len(nodes))
    return {"aggregate": d["aggregate"], "nodes": nodes, "expected_nodes": expected,
            "diagnosis": {"primary": d["primary"], "issues": d["issues"]}}


# ----------------------------------------------------------------------------- driver
class SummaryEngine:
    """All three sections for the local engines of this process."""

    def __init__(self, engines, comm=None, *, exchange: str = "auto",
                 ram_total: Optional[float] = None, gpu_count: Optional[int] = None, native: bool = True,
                 system_identity: Optional[Dict[str, Any]] = None):
        self.reducer = WindowReducer(engines, comm, exchange=exchange, native=native)
        self.engines = list(engines)
        self.comm = self.reducer.comm
        if ram_total is None:
            try:
                import psutil

                ram_total = float(psutil.virtual_memory().total)
            except Exception:
                ram_total = float(os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES"))
        self.ram_total = ram_total
        self.gpu_count = gpu_count
        self._unemitted: Optional[_abi.Sections] = None  # the last native build's sections
        self._sec_key = None  # the sections' args, shared by builds with the same values
        self._sec_args: Optional[_abi.SectionsArgs] = None
        # the System section has one source per node: the engine of local rank 0, whose system
        # ring the sampler fills; its node identity comes from the launcher's environment.  On one
        # node that is comm index 0; on several, every node leader reduces its own ring and the
        # records meet on comm index 0 (multi_node_run).
        self.system_identity = system_identity
        self._ident: Optional[Dict[str, Any]] = None
        self._no_system: Optional[Dict[str, Any]] = None
        self.multi_node = multi_node_run(self.comm)
        self._node_ident: Optional[Dict[str, Any]] = None

    def _leader_identity(self) -> Dict[str, Any]:
        if self._node_ident is None:
            from .reporting import default_identity

            self._node_ident = self.system_identity or default_identity(
                self.comm.index, max(1, int(self.comm.world)) * max(1, len(self.engines)))
        return self._node_ident

    def _system_launch(self, rows: int):
        """K6s beside the window pass on the engine holding the system ring; None (and nothing
        launched) when this process is not its node's source or its ring is empty."""
        eng = self.engines[0] if self.engines else None
        if self.multi_node:
            source = int(self._leader_identity().get("local_rank") or 0) == 0
        else:
            source = self.comm.index == 0
        if not source or not hasattr(eng, "sys_reduce_beside") or eng.sys_count == 0:
            return None
        eng.sys_reduce_beside(rows, _stream_of(self.reducer.device))
        return eng

    def _system_gather(self, eng) -> Optional[Dict[str, Any]]:
        """Every rank packs its node record in device memory (valid only on a node leader with
        samples); one all-gather brings them to comm index 0, which folds them (K6m), copies the
        records and the cluster rollup back in one transfer and runs the cluster rules.  None on
        every other rank."""
        import ctypes as C

        import torch

        if eng is not None:
            eng.sys_reduce_collect()  # ends the launch; the node's aggregates stay in HBM for the pack
        dev, world = self.reducer.device, int(self.comm.world)
        rec = C.sizeof(_abi.SysNodeRecord)
        mine = torch.empty(rec, dtype=torch.uint8, device=dev)
        gathered = torch.empty(world * rec + C.sizeof(_abi.SysClusterOut), dtype=torch.uint8, device=dev)
        stream = _stream_of(dev)
        ident = node_ident(self._leader_identity()) if eng is not None else None
        self.engines[0].sys_node_pack(ident, mine, stream)
        self.comm.all_gather_into(gathered[: world * rec], mine)
        if self.comm.index != 0:
            return None
        self.engines[0].sys_cluster_launch(gathered, world, stream)
        records, cluster = self.engines[0].sys_cluster_collect(world)
        if cluster.n_dup:
            import sys

            print(f"[TraceML] System section: {int(cluster.n_dup)} node record(s) repeat a node label; "
                  "each label keeps the record of its lowest global rank", file=sys.stderr)
        return build_system_cluster(records, cluster)

    def _system_section(self, eng) -> Optional[Dict[str, Any]]:
        if self.multi_node:
            return self._system_gather(eng)
        if self._ident is None:
            from .reporting import default_identity

            self._ident = self.system_identity or default_identity(
                0, max(1, int(self.comm.world)) * max(1, len(self.engines)))
        if eng is None:  # zero samples (NO_DATA): the same section every build
            if self._no_system is None:
                self._no_system = build_system(None, self._ident)
            return self._no_system
        return build_system(eng.sys_reduce_collect(), self._ident)

    def build(self, window: int = 10_000, proc_rows: int = 10_000, *, timings: bool = False) -> _abi.Sections:
        import torch

        gpu_count = self.gpu_count if self.gpu_count is not None else torch.cuda.device_count()
        rows = max(1, int(proc_rows))
        w = max(1, int(window))
        native = self.reducer._native_ok() and not timings
        seng = self._system_launch(rows)  # K6s beside the window pass; nothing without samples
        if native:
            # one rank per process: stages, exchanges and rule engines all native (csrc/tml_summary.cpp).
            # The driver writes into a struct the result owns, so nothing is copied after the wait.
            # The text is emitted from that struct: on first access, or by the next build while its
            # window pass runs, whichever comes first -- so back-to-back builds keep the JSON
            # emitter out of the time the GPU waits for the host.
            prev = self._unemitted
            o = self.reducer.run_native(w, rows, prev=prev if prev is not None and prev._raw is None else None,
                                        out=_abi.ReduceRunOut())
            red = self.reducer.native_result(o, w, owned=True)
        else:
            red = self.reducer.reduce(w, proc_rows=rows, stage_timings=timings)
        # ram_total / gpu_count are per-host constants (psutil.virtual_memory().total,
        # torch.cuda.device_count()); single-node scope: identical on every rank.  The emitter only
        # reads its args, so builds with the same values share one struct.
        key = (self.ram_total, gpu_count, w, rows)
        if key != self._sec_key:
            self._sec_args = _abi.SectionsArgs(float(self.ram_total), int(gpu_count), w, rows, 0)
            self._sec_key = key
        res = _abi.Sections(src=red.out, args=self._sec_args)
        res["reduce"] = red
        res["system"] = self._system_section(seng)
        if native:
            self._unemitted = res
        return res


__all__ = ["SummaryEngine", "build_process", "build_system", "build_system_cluster", "multi_node_run",
           "node_ident", "proc_agg_dict", "system_node_label"]
