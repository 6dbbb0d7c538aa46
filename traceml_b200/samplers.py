"""Sampler-side views: device records -> the reference's wire rows.

Replaces ``StepTimeSampler`` / ``StepMemorySampler`` / ``ProcessSampler``
(``src/traceml/samplers/{step_time,step_memory,process}_sampler.py``).  The
step samplers become a drain of the host-mapped record mirror (no CUDA call,
no event queries); the process sampler still reads CPU% / RSS on the host
(psutil) but commits the sample through ``tml_proc_commit`` into the device
proc ring so the Process reduce runs on the GPU with the rest.
"""
from __future__ import annotations

import os
import time
from typing import Any, Dict, List, Optional

from .records import (PROC_FLAG_GPU_AVAILABLE, PROC_FLAG_HAS_GPU_METRICS, proc_record_to_wire,
                      step_record_to_memory_wire, step_record_to_wire)


_HOST_CONSTS: Dict[str, Any] = {}


def host_constants() -> Dict[str, Any]:
    """Per-host constants of a process wire row (samplers/process_sampler.py:96-123):
    ``ram_total`` = psutil.virtual_memory().total, ``gpu_count`` = torch.cuda.device_count().
    Read once; they are not in the 64-B device record."""
    if not _HOST_CONSTS:
        try:
            import psutil

            _HOST_CONSTS["ram_total"] = float(psutil.virtual_memory().total)
        except Exception:
            _HOST_CONSTS["ram_total"] = float(os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES"))
        try:
            import torch

            _HOST_CONSTS["gpu_count"] = int(torch.cuda.device_count()) if torch.cuda.is_available() else 0
        except Exception:
            _HOST_CONSTS["gpu_count"] = 0
    return _HOST_CONSTS


def drain_to_wire(engine, device: Optional[str] = None, ram_total: Optional[float] = None,
                  gpu_count: Optional[int] = None) -> Dict[str, Any]:
    """Completed records since the last call as wire rows
    (samplers/schema/step_time_schema.py:85-96, step_memory.py:41-58, process.py:139-150)."""
    dev = device or f"cuda:{engine.device}"
    recs, dropped = engine.drain()
    procs, pdropped = engine.proc_drain()
    now = time.time()
    if procs is not None and len(procs) and (ram_total is None or gpu_count is None):
        hc = host_constants()
        ram_total = hc["ram_total"] if ram_total is None else ram_total
        gpu_count = hc["gpu_count"] if gpu_count is None else gpu_count
    return {
        "step_time": [step_record_to_wire(r, device=dev) for r in recs],
        "step_memory": [step_record_to_memory_wire(r, device=dev, ts=now) for r in recs],
        "process": [proc_record_to_wire(p, pid=os.getpid(), device_index=engine.device,
                                        ram_total=float(ram_total or 0.0), gpu_count=int(gpu_count or 0))
                    for p in procs],
        "dropped": int(dropped) + int(pdropped),
    }


class ProcessProbe:
    """One process sample per call (samplers/process_sampler.py:178-238)."""

    def __init__(self):
        import psutil

        self.proc = psutil.Process(os.getpid())
        self.proc.cpu_percent(interval=None)  # warm-up, as the reference does
        self.cores = psutil.cpu_count(logical=True) or 0
        self.ram_total = float(psutil.virtual_memory().total)
        self.seq = 0
        self._stream = None
        self._total = None

    def _cuda_safe(self) -> bool:
        # never touch CUDA before dist.init_process_group() in a distributed job
        # (process_sampler.py:150-158)
        if int(os.environ.get("WORLD_SIZE", "1") or 1) <= 1:
            return True
        try:
            import torch.distributed as dist

            return dist.is_available() and dist.is_initialized()
        except Exception:
            return False

    def sample(self, engine) -> None:
        import torch

        from .utils.step_memory import _alloc_ext

        self.seq += 1
        cpu = float(self.proc.cpu_percent(interval=None))
        rss = int(self.proc.memory_info().rss)
        flags, used, resv, total = 0, 0, 0, 0
        if self._cuda_safe() and torch.cuda.is_available():
            flags |= PROC_FLAG_GPU_AVAILABLE | PROC_FLAG_HAS_GPU_METRICS
            ext = _alloc_ext()
            if ext is not None:
                used, resv = ext.current_bytes(engine.device)
            else:
                used = torch.cuda.memory_allocated(engine.device)
                resv = torch.cuda.memory_reserved(engine.device)
            if self._total is None:
                self._total = int(torch.cuda.get_device_properties(engine.device).total_memory)
            total = self._total
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=engine.device)  # side stream, never the training stream
        engine.proc_commit(self.seq, time.time(), cpu, rss, int(used), int(resv), int(total), flags,
                           int(self.cores), int(self._stream.cuda_stream))


# ----------------------------------------------------------------------------- sampler seam
class TableStore:
    """The table contract of ``database/database.py:7-186``: bounded ``deque(maxlen=3000)``
    per table plus a monotonic append counter, so the kept incremental sender can find the
    new rows in O(1)."""

    DEFAULT_MAX_ROWS = 3000

    def __init__(self, sampler_name: str, max_rows: Optional[int] = None):
        from collections import deque

        self.sampler_name = sampler_name
        self.max_rows = int(max_rows) if max_rows is not None else self.DEFAULT_MAX_ROWS
        if self.max_rows <= 0:
            raise ValueError(f"max_rows must be > 0, got {max_rows}")
        self._deque = deque
        self._tables: Dict[str, Any] = {}
        self._append_count: Dict[str, int] = {}

    def create_or_get_table(self, name: str):
        if name not in self._tables:
            self._tables[name] = self._deque(maxlen=self.max_rows)
            self._append_count[name] = 0
        return self._tables[name]

    def add_record(self, table: str, row: Any) -> None:
        self.create_or_get_table(table).append(row)
        self._append_count[table] += 1

    def all_tables(self) -> Dict[str, Any]:
        return self._tables

    def get_append_count(self, table: str) -> int:
        return self._append_count.get(table, 0)


def _identity_fields() -> Dict[str, Any]:
    """database/database_sender.py:49-66 envelope identity, from the launcher's env contract."""
    import socket

    rank = int(os.environ.get("RANK", "0") or 0)
    return {
        "rank": rank, "global_rank": rank,
        "local_rank": int(os.environ.get("LOCAL_RANK", "0") or 0),
        "world_size": int(os.environ.get("WORLD_SIZE", "1") or 1),
        "local_world_size": int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1")) or 1),
        "node_rank": int(os.environ.get("GROUP_RANK", os.environ.get("NODE_RANK", "0")) or 0),
        "hostname": socket.gethostname(), "pid": os.getpid(),
    }


class RecordTap:
    """One drain cursor per engine, fanned out: the step-time and step-memory samplers read
    the same 128-B records."""

    def __init__(self, engine):
        self.engine = engine
        self.pending: Dict[str, List[Any]] = {"step_time": [], "step_memory": [], "process": []}
        self.dropped = 0

    def pump(self) -> None:
        out = drain_to_wire(self.engine)
        self.dropped += out["dropped"]
        for k in self.pending:
            self.pending[k].extend(out[k])

    def take(self, kind: str) -> List[Any]:
        rows, self.pending[kind] = self.pending[kind], []
        return rows


class _TapSampler:
    """``BaseSampler`` contract (samplers/base_sampler.py:23-83): ``sampler_name``,
    ``table_name``, ``db``, ``sample()`` that never raises, and ``collect_payload()`` with the
    sender's envelope (database/database_sender.py:127-170)."""

    sampler_name = ""
    table_name = ""
    kind = ""

    def __init__(self, tap: RecordTap, max_rows_per_flush: int = -1):
        self.tap = tap
        self.db = TableStore(self.sampler_name)
        self.max_rows_per_flush = int(max_rows_per_flush)
        self.enable_send = True
        self._last_sent: Dict[str, int] = {}

    def sample(self) -> None:
        try:
            self.tap.pump()
            for row in self.tap.take(self.kind):
                self.db.add_record(self.table_name, row)
        except Exception as exc:  # noqa: BLE001 -- samplers never interfere with training
            import sys

            print(f"[TraceML] {self.sampler_name}.sample failed: {exc}", file=sys.stderr)

    def collect_payload(self) -> Optional[Dict[str, Any]]:
        tables: Dict[str, List[Any]] = {}
        for name, rows in self.db.all_tables().items():
            total = self.db.get_append_count(name)
            new = total - self._last_sent.get(name, 0)
            if not rows or new <= 0:
                continue
            if self.max_rows_per_flush != -1:
                new = min(new, self.max_rows_per_flush)
            n = len(rows)
            tables[name] = list(rows) if new >= n else [rows[i] for i in range(n - new, n)]
            self._last_sent[name] = total
        if not tables:
            return None
        return {**_identity_fields(), "sampler": self.sampler_name, "timestamp": time.time(), "tables": tables}


class StepTimeSampler(_TapSampler):
    """samplers/step_time_sampler.py:21-128 -- a drain of finished records, no event queries."""
    sampler_name, table_name, kind = "StepTimeSampler", "StepTimeTable", "step_time"


class StepMemorySampler(_TapSampler):
    """samplers/step_memory_sampler.py:12-65."""
    sampler_name, table_name, kind = "StepMemorySampler", "step_memory", "step_memory"


class ProcessSampler(_TapSampler):
    """samplers/process_sampler.py:36-238 -- takes a sample (host CPU / RSS + allocator counters,
    committed to the device ring), then publishes what the ring produced."""
    sampler_name, table_name, kind = "ProcessSampler", "ProcessTable", "process"

    def __init__(self, tap: RecordTap, max_rows_per_flush: int = -1, probe: Optional[ProcessProbe] = None):
        super().__init__(tap, max_rows_per_flush)
        self.probe = probe

    def sample(self) -> None:
        try:
            if self.probe is None:
                self.probe = ProcessProbe()
            self.probe.sample(self.tap.engine)
        except Exception as exc:  # noqa: BLE001
            import sys

            print(f"[TraceML] ProcessSampler probe failed: {exc}", file=sys.stderr)
        super().sample()


class SystemProbe:
    """One host / all-GPU snapshot per call: the wire row of ``SystemSample.to_wire``
    (samplers/system_sampler.py:42-221, samplers/schema/system.py:133-157) and the same snapshot
    as the engine's fixed-size system record (the raw NVML integers; watts are derived from them
    as ``mW / 1000.0`` exactly where the wire row does it).  Host-side by nature (psutil + NVML).
    NVML failures degrade to CPU/RAM only, a failing GPU yields the reference's zeroed placeholder
    so that index == GPU id.  The record keeps the first 16 GPUs of a host."""

    def __init__(self):
        import psutil

        self._psutil = psutil
        self.seq = 0
        self.cores = 0
        self.ram_total = 0.0
        self.gpu_available = False
        self.gpu_count = 0
        self._nvml = None
        self._handles: Dict[int, Any] = {}
        try:
            psutil.cpu_percent(interval=None)  # warm-up: the first real call must not block
            self.cores = psutil.cpu_count(logical=True) or 0
            self.ram_total = float(psutil.virtual_memory().total)
        except Exception:
            pass
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nvml = pynvml
            self.gpu_count = int(pynvml.nvmlDeviceGetCount())
            self.gpu_available = self.gpu_count > 0
        except Exception:
            self._nvml = None

    def _raw_gpus(self) -> List[tuple]:
        """(util %, mem used, mem total, temp C, power mW, power limit mW) per GPU, as NVML
        returns them; zeros for a GPU whose query failed."""
        if not self.gpu_available or self._nvml is None:
            return []
        n, out = self._nvml, []
        for i in range(self.gpu_count):
            try:
                h = self._handles.get(i)
                if h is None:  # a handle is fixed for the process: looked up once (again after a failure)
                    h = self._handles[i] = n.nvmlDeviceGetHandleByIndex(i)
                util = n.nvmlDeviceGetUtilizationRates(h)
                mem = n.nvmlDeviceGetMemoryInfo(h)
                temp = n.nvmlDeviceGetTemperature(h, n.NVML_TEMPERATURE_GPU)
                out.append((int(util.gpu), int(mem.used), int(mem.total), int(temp),
                            int(n.nvmlDeviceGetPowerUsage(h)), int(n.nvmlDeviceGetPowerManagementLimit(h))))
            except Exception:
                out.append((0, 0, 0, 0, 0, 0))
        return out

    def _gpus(self) -> List[List[float]]:
        return [self._wire_gpu(g) for g in self._raw_gpus()]

    @staticmethod
    def _wire_gpu(g: tuple) -> List[float]:
        util, used, total, temp, mw, limit_mw = g
        return [float(util), float(used), float(total), float(temp), float(mw / 1000.0), float(limit_mw / 1000.0)]

    def snapshot(self):
        """(wire row, ``_abi.SysRecord``) of one sample: the same numbers twice."""
        self.seq += 1
        try:
            cpu = float(self._psutil.cpu_percent(interval=None))
        except Exception:
            cpu = 0.0
        try:
            ram_used = int(self._psutil.virtual_memory().used)
        except Exception:
            ram_used = 0
        ts = time.time()
        raw = self._raw_gpus()
        row = {"seq": self.seq, "ts": ts, "cpu": cpu, "ram_used": float(ram_used),
               "ram_total": self.ram_total, "gpu_available": self.gpu_available,
               "gpu_count": self.gpu_count, "gpus": [self._wire_gpu(g) for g in raw]}
        return row, sys_record(self.seq, ts, cpu, ram_used, int(self.ram_total), self.gpu_available,
                               self.gpu_count, raw)

    def sample(self) -> Dict[str, Any]:
        return self.snapshot()[0]


def sys_record(seq: int, ts: float, cpu: float, ram_used: int, ram_total: int, gpu_available: bool,
               gpu_count: int, gpus) -> Any:
    """The engine's 576-B system record of one snapshot; ``gpus`` = raw NVML integer tuples
    (util %, mem used, mem total, temp C, power mW, power limit mW), the first 16 kept."""
    from . import _abi

    r = _abi.SysRecord()
    r.seq, r.ts, r.cpu_pct, r.ram_used, r.ram_total = int(seq), float(ts), float(cpu), int(ram_used), int(ram_total)
    r.flags = _abi.SYS_GPU_AVAILABLE if gpu_available else 0
    r.gpu_count = int(gpu_count)
    gpus = list(gpus)[: _abi.TML_SYS_MAX_GPUS]
    r.n_gpus = len(gpus)
    for i, (util, used, total, temp, mw, limit_mw) in enumerate(gpus):
        e = r.gpu[i]
        e.util, e.mem_used, e.mem_total, e.temp_c = int(util), int(used), int(total), int(temp)
        e.power_mw, e.power_limit_mw = int(mw), int(limit_mw)
    return r


class SystemSampler:
    """``BaseSampler`` contract for the host snapshot (runtime/sampler_registry.py:78-105:
    ``system``, rank-zero only, ``max_rows_per_flush=1``)."""

    sampler_name, table_name, kind = "SystemSampler", "SystemTable", "system"

    def __init__(self, probe: Optional[SystemProbe] = None):
        self.probe = probe
        self.db = TableStore(self.sampler_name)
        self.max_rows_per_flush = 1
        self.enable_send = True
        self._last_sent: Dict[str, int] = {}

    def sample(self) -> None:
        try:
            if self.probe is None:
                self.probe = SystemProbe()
            self.db.add_record(self.table_name, self.probe.sample())
        except Exception as exc:  # noqa: BLE001
            import sys

            print(f"[TraceML] SystemSampler.sample failed: {exc}", file=sys.stderr)

    collect_payload = _TapSampler.collect_payload


def build_samplers(engine, rank_zero: Optional[bool] = None) -> List[Any]:
    """The per-rank sampler set of profile ``run`` that is on this path
    (runtime/sampler_registry.py:78-160: system on local rank 0; process, step_time, step_memory
    on every rank)."""
    tap = RecordTap(engine)
    out: List[Any] = []
    if rank_zero is None:
        rank_zero = int(os.environ.get("LOCAL_RANK", "0") or 0) == 0
    if rank_zero:
        out.append(SystemSampler())
    return out + [ProcessSampler(tap), StepTimeSampler(tap), StepMemorySampler(tap)]


__all__ = ["drain_to_wire", "ProcessProbe", "SystemProbe", "sys_record", "TableStore", "RecordTap", "StepTimeSampler",
           "StepMemorySampler", "ProcessSampler", "SystemSampler", "build_samplers", "host_constants"]
