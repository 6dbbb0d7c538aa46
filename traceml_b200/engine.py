"""Per-GPU engine handle: a thin object wrapper over the C-ABI context.

One ``Engine`` per (process, GPU) -- the GPU-native replacement for the
reference's per-rank ``TraceMLRuntime`` + queues + samplers
(``src/traceml/runtime/runtime.py:33-193``).  Tests may create several engines
on one GPU to play several ranks.
"""

from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import numpy as np

from . import _abi
from .records import PROC_RECORD_DTYPE, STEP_RECORD_DTYPE


def _p(x) -> int:
    """Raw device address of a torch tensor (or pass an int through)."""
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x or 0)


class _DevView:
    """Zero-copy torch view of device memory owned by the native library."""

    def __init__(self, ptr: int, n_f64: int):
        self.__cuda_array_interface__ = {
            "shape": (int(n_f64),), "typestr": "<f8", "data": (int(ptr), False), "version": 2,
        }


class Engine:
    def __init__(self, device: int = 0, rank: int = 0, world: int = 1,
                 ring_slots: int = 15_000, proc_slots: int = 15_000):
        self._lib = _abi.lib()
        self.device, self.rank, self.world = int(device), int(rank), int(world)
        self.ring_slots, self.proc_slots = int(ring_slots), int(proc_slots)
        h = C.c_void_p()
        _abi.check(self._lib.tml_init(self.device, self.rank, self.world, self.ring_slots,
                                      self.proc_slots, C.byref(h)), "tml_init")
        self._h = h
        # bound C functions for the step path (attribute lookups are not free)
        self._begin = self._lib.tml_phase_begin
        self._end = self._lib.tml_phase_end
        self._host = self._lib.tml_phase_host
        self._commit = self._lib.tml_step_commit
        self._drain_buf = np.zeros(4096, dtype=STEP_RECORD_DTYPE)
        self._pdrain_buf = np.zeros(8192, dtype=PROC_RECORD_DTYPE)
        self._run_out = _abi.ReduceRunOut()

    # ------------------------------------------------------------ lifecycle
    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            # the step glue / native sampler hold this context's raw pointer: unbind them first
            import sys

            timing = sys.modules.get("traceml_b200.utils.timing")
            if timing is not None and getattr(timing, "_ENG", None) is self:
                timing._reset()
            self._lib.tml_shutdown(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # best effort
        try:
            self.close()
        except Exception:
            pass

    def reset(self) -> None:
        _abi.check(self._lib.tml_ring_reset(self._h), "tml_ring_reset")

    # ------------------------------------------------------------ step path
    def phase_begin(self, phase: int, stream: int) -> int:
        return self._begin(self._h, phase, stream)

    def phase_end(self, phase: int, slot: int, stream: int) -> int:
        return self._end(self._h, phase, slot, stream)

    def phase_host(self, phase: int, dur_ns: int) -> int:
        return self._host(self._h, phase, dur_ns)

    def step_commit(self, step: int, peak_alloc: int, peak_resv: int, flags: int,
                    host_ts: float, stream: int) -> int:
        return self._commit(self._h, step, peak_alloc, peak_resv, flags, host_ts, stream)

    def step_discard(self) -> None:
        self._lib.tml_step_discard(self._h)

    @property
    def step_count(self) -> int:
        return int(self._lib.tml_step_count(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._lib.tml_launch_count(self._h))

    @property
    def proc_count(self) -> int:
        return int(self._lib.tml_proc_count(self._h))

    # ------------------------------------------------------------ sampler side
    def drain(self) -> Tuple[np.ndarray, int]:
        """Completed StepRecords since the last drain (no CUDA call)."""
        n, dropped = C.c_uint32(0), C.c_uint64(0)
        out = []
        while True:
            _abi.check(self._lib.tml_drain(self._h, self._drain_buf.ctypes.data,
                                           len(self._drain_buf), C.byref(n), C.byref(dropped)),
                       "tml_drain")
            if n.value:
                out.append(self._drain_buf[: n.value].copy())
            if n.value < len(self._drain_buf):
                break
        recs = np.concatenate(out) if out else np.zeros(0, dtype=STEP_RECORD_DTYPE)
        return recs, int(dropped.value)

    def proc_drain(self) -> Tuple[np.ndarray, int]:
        n, dropped = C.c_uint32(0), C.c_uint64(0)
        out = []
        while True:
            _abi.check(self._lib.tml_proc_drain(self._h, self._pdrain_buf.ctypes.data,
                                                len(self._pdrain_buf), C.byref(n),
                                                C.byref(dropped)), "tml_proc_drain")
            if n.value:
                out.append(self._pdrain_buf[: n.value].copy())
            if n.value < len(self._pdrain_buf):
                break
        recs = np.concatenate(out) if out else np.zeros(0, dtype=PROC_RECORD_DTYPE)
        return recs, int(dropped.value)

    def live(self) -> _abi.LiveStats:
        out = _abi.LiveStats()
        _abi.check(self._lib.tml_live(self._h, C.byref(out)), "tml_live")
        return out

    def proc_commit(self, seq: int, ts: float, cpu_pct: float, rss: int, mem_alloc: int,
                    mem_resv: int, mem_total: int, flags: int, cpu_cores: int,
                    stream: int = 0) -> None:
        r = _abi.ProcRecord(seq, ts, cpu_pct, rss, mem_alloc, mem_resv, mem_total, flags, cpu_cores)
        _abi.check(self._lib.tml_proc_commit(self._h, C.byref(r), stream), "tml_proc_commit")

    def load_steps(self, records: np.ndarray, stream: int = 0) -> None:
        """Bulk-append StepRecords from host memory (async H2D on ``stream``)."""
        records = np.ascontiguousarray(records, dtype=STEP_RECORD_DTYPE)
        self._keep = records  # keep alive until the stream is synchronised
        _abi.check(self._lib.tml_ring_load(self._h, records.ctypes.data, len(records), stream),
                   "tml_ring_load")

    def load_steps_ptr(self, host_ptr: int, n: int, stream: int = 0) -> None:
        _abi.check(self._lib.tml_ring_load(self._h, host_ptr, n, stream), "tml_ring_load")

    def load_procs(self, records: np.ndarray, stream: int = 0) -> None:
        records = np.ascontiguousarray(records, dtype=PROC_RECORD_DTYPE)
        self._keep_p = records
        _abi.check(self._lib.tml_proc_load(self._h, records.ctypes.data, len(records), stream),
                   "tml_proc_load")

    # ------------------------------------------------------------ reduce stages
    def win_prepare(self, window: int, stream: int = 0) -> _abi.WinInfo:
        out = _abi.WinInfo()
        _abi.check(self._lib.tml_win_prepare(self._h, int(window), stream, C.byref(out)),
                   "tml_win_prepare")
        return out

    def win_presence(self, kind: int, glo: int, span: int, presence, stream: int = 0) -> None:
        _abi.check(self._lib.tml_win_presence(self._h, kind, glo, span, _p(presence), stream),
                   "tml_win_presence")

    def win_select(self, kind: int, glo: int, span: int, presence, window: int,
                   stream: int = 0) -> _abi.AlignInfo:
        out = _abi.AlignInfo()
        _abi.check(self._lib.tml_win_select(self._h, kind, glo, span, _p(presence), int(window),
                                            stream, C.byref(out)), "tml_win_select")
        return out

    def win_select_dense(self, kind: int, first_step: int, n_common: int,
                         stream: int = 0) -> _abi.AlignInfo:
        out = _abi.AlignInfo()
        _abi.check(self._lib.tml_win_select_dense(self._h, kind, int(first_step), int(n_common),
                                                  stream, C.byref(out)), "tml_win_select_dense")
        return out

    def win_rows_ptr(self, kind: int) -> int:
        return int(self._lib.tml_win_rows(self._h, kind) or 0)

    def win_rows_tensor(self, kind: int, n_common: int):
        """This rank's aligned rows as a flat f64 torch tensor (no copy)."""
        import torch

        ptr = self.win_rows_ptr(kind)
        if not ptr or n_common <= 0:
            return torch.empty(0, dtype=torch.float64, device=f"cuda:{self.device}")
        return torch.as_tensor(_DevView(ptr, n_common * 8), device=f"cuda:{self.device}")

    def win_rows_export(self, kind: int) -> bytes:
        """72 bytes: the 64-B CUDA-IPC handle of the allocation + the rows' byte offset."""
        buf = C.create_string_buffer(64)
        off = C.c_uint64(0)
        _abi.check(self._lib.tml_win_rows_export(self._h, kind, buf, C.byref(off)),
                   "tml_win_rows_export")
        return bytes(buf.raw) + int(off.value).to_bytes(8, "little")

    def peer_open(self, handle: bytes) -> int:
        p = C.c_void_p()
        _abi.check(self._lib.tml_peer_open(self._h, handle[:64], C.byref(p)), "tml_peer_open")
        return int(p.value) + int.from_bytes(handle[64:72], "little")

    def reduce_run(self, window: int, proc_rows: int, exchange: str, speculate: bool, comm_ptr: int,
                   rank: int, world: int, stream: int = 0) -> _abi.ReduceRunOut:
        """The whole staged reduce, sequenced natively (csrc/tml_summary.cpp)."""
        comm = _abi.Comm(comm_ptr or None, int(rank), int(world))
        args = _abi.ReduceRunArgs(int(window), int(proc_rows or 0), _abi.XCHG[exchange], 1 if speculate else 0)
        out = self._run_out  # ~45 KB: reused, not reallocated per call
        _abi.check(self._lib.tml_reduce_run(self._h, C.byref(comm), C.byref(args), stream, C.byref(out)),
                   "tml_reduce_run")
        return out

    def sections_json(self, run_out, ram_total: float, gpu_count: int, window: int, proc_rows: int):
        """Step-Time / Step-Memory / Process sections of a reduce_run, parsed (csrc/tml_sections.cpp)."""
        return _abi.sections_json(run_out, ram_total, gpu_count, window, proc_rows)

    def kernel_ms(self, which: int) -> float:
        """Device time of the last K3a (0) / K4 (1) launch, from the library's own events."""
        return float(self._lib.tml_kernel_ms(self._h, int(which)))

    # ---- live tick (StepCombined / step-memory combined twins): header "LIVE TICK"
    def combined_prepare(self, kind: int, lookback: int, stream: int = 0) -> _abi.CombinedInfo:
        out = _abi.CombinedInfo()
        _abi.check(self._lib.tml_combined_prepare(self._h, kind, int(lookback), stream, C.byref(out)),
                   "tml_combined_prepare")
        return out

    def combined_presence(self, kind: int, glo: int, span: int, presence, stream: int = 0) -> None:
        _abi.check(self._lib.tml_combined_presence(self._h, kind, int(glo), int(span), _p(presence),
                                                   stream), "tml_combined_presence")

    def combined_select(self, kind: int, glo: int, span: int, presence, window: int,
                        stream: int = 0) -> _abi.CombinedAlign:
        out = _abi.CombinedAlign()
        _abi.check(self._lib.tml_combined_select(self._h, kind, int(glo), int(span), _p(presence),
                                                 int(window), stream, C.byref(out)), "tml_combined_select")
        return out

    def combined_rows_ptr(self, kind: int) -> int:
        return int(self._lib.tml_combined_rows(self._h, kind) or 0)

    def combined_rows_tensor(self, kind: int, n_common: int):
        import torch

        ptr = self.combined_rows_ptr(kind)
        if not ptr or n_common <= 0:
            return torch.empty(0, dtype=torch.float64, device=f"cuda:{self.device}")
        return torch.as_tensor(_DevView(ptr, n_common * 8), device=f"cuda:{self.device}")

    def combined_steps(self, kind: int, n_common: int, stream: int = 0):
        buf = (C.c_uint64 * max(1, int(n_common)))()
        _abi.check(self._lib.tml_combined_steps(self._h, kind, buf, int(n_common), stream),
                   "tml_combined_steps")
        return [int(buf[i]) for i in range(int(n_common))]

    def combined_series(self, row_ptrs, n_common: int, first_col: int, n_cols: int, series,
                        stream: int = 0) -> None:
        arr = (C.c_void_p * len(row_ptrs))(*[int(p) for p in row_ptrs])
        _abi.check(self._lib.tml_combined_series(self._h, arr, len(row_ptrs), int(n_common), int(first_col),
                                                 int(n_cols), _p(series), stream), "tml_combined_series")

    def win_reduce(self, rows, mask: int, n_common: int, shard_lo: int,
                   shard_hi: int, series, stream: int = 0) -> None:
        a = _abi.ReduceArgs()
        a.n_ranks, a.mask, a.n_common = len(rows), mask, n_common
        a.shard_lo, a.shard_hi, a.series = shard_lo, shard_hi, _p(series)
        for i, p in enumerate(rows):
            a.rows[i] = _p(p)
        _abi.check(self._lib.tml_win_reduce(self._h, C.byref(a), stream), "tml_win_reduce")

    def win_bands(self, series, args: _abi.BandArgs, stream: int = 0) -> _abi.BandOut:
        out = _abi.BandOut()
        _abi.check(self._lib.tml_win_bands(self._h, _p(series), C.byref(args), stream,
                                           C.byref(out)), "tml_win_bands")
        return out

    def proc_reduce_launch(self, max_rows: int, stream: int = 0) -> None:
        _abi.check(self._lib.tml_proc_reduce_launch(self._h, int(max_rows), stream),
                   "tml_proc_reduce_launch")

    def proc_reduce_collect(self) -> _abi.ProcAgg:
        out = _abi.ProcAgg()
        _abi.check(self._lib.tml_proc_reduce_collect(self._h, C.byref(out)), "tml_proc_reduce_collect")
        return out

    def proc_reduce(self, max_rows: int, stream: int = 0) -> _abi.ProcAgg:
        out = _abi.ProcAgg()
        _abi.check(self._lib.tml_proc_reduce(self._h, int(max_rows), stream, C.byref(out)),
                   "tml_proc_reduce")
        return out


__all__ = ["Engine"]
