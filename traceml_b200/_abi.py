"""ctypes binding of ``libtraceml_b200.so`` (declared in ``include/traceml_b200.h``).

This is the only place Python crosses into native code.  Loading fails loudly:
there is no pure-Python or CPU fallback for any entry point.
"""

from __future__ import annotations

import ctypes as C
import json
import os
from typing import Any, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtraceml_b200.so")

TML_N_PHASES = 6
TML_MAX_PHASES = 8
TML_MAX_RANKS = 64
TML_SERIES_PER_STEP = 16
TML_OK = 0
TML_ERR_CAPTURE = -7
TML_ERR_NONMONOTONIC = -5
KIND_TIME, KIND_MEM = 0, 1
MASK_TIME, MASK_MEM = 1, 2

u8, u32, u64, i32, i64, f64 = C.c_uint8, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_double
vp = C.c_void_p


class StepRecord(C.Structure):
    _fields_ = [("step", u64), ("dur_ns", u64 * TML_N_PHASES), ("n_calls", u32 * TML_N_PHASES),
                ("peak_alloc", u64), ("peak_resv", u64), ("host_ts", f64), ("gpu_mask", u32),
                ("flags", u32), ("seq", u64), ("_pad", u64)]


class ProcRecord(C.Structure):
    _fields_ = [("seq", u64), ("ts", f64), ("cpu_pct", f64), ("rss", u64), ("mem_alloc", u64),
                ("mem_resv", u64), ("mem_total", u64), ("flags", u32), ("cpu_cores", u32)]


class LayerRecord(C.Structure):
    _fields_ = [("step", u64), ("fwd_ns", u64), ("bwd_ns", u64), ("fwd_calls", u32), ("bwd_calls", u32),
                ("fwd_bytes", u64), ("bwd_bytes", u64)]


class LivePhase(C.Structure):
    _fields_ = [("count", u64), ("sum_ns", u64), ("worst_ns", u64), ("median_ns", u64)]


class LiveStats(C.Structure):
    _fields_ = [("steps_committed", u64), ("phase", LivePhase * TML_MAX_PHASES)]


class WinInfo(C.Structure):
    _fields_ = [("n_retained", u64), ("latest_step", u64), ("monotone", u32), ("dup_rows", u32),
                ("n_rows", u64 * 2), ("n_cand", u64 * 2), ("lo", u64 * 2), ("hi", u64 * 2),
                ("t_sums", f64 * 7), ("t_count", u64), ("n_both", u64), ("dense", u32 * 2), ("kernel_ms", f64)]


class AlignInfo(C.Structure):
    _fields_ = [("n_common", u64), ("start_step", u64), ("end_step", u64), ("n_rows", u64),
                ("t_sums", f64 * 7), ("m_sums", f64 * 4)]


class CombinedInfo(C.Structure):
    _fields_ = [("n_rows", u64), ("n_cand", u64), ("lo", u64), ("hi", u64), ("latest_step", u64),
                ("first_step", u64), ("truncated", u32), ("monotone", u32)]


class CombinedAlign(C.Structure):
    _fields_ = [("n_common", u64), ("n_rows", u64), ("sums", f64 * 6), ("peaks", f64 * 2)]


class ReduceArgs(C.Structure):
    _fields_ = [("n_ranks", u32), ("mask", u32), ("n_common", u64), ("shard_lo", u64),
                ("shard_hi", u64), ("rows", vp * TML_MAX_RANKS), ("series", vp)]


class BandArgs(C.Structure):
    _fields_ = [("n_common", u64), ("shard_lo", u64), ("shard_hi", u64),
                ("band_lo", (u64 * 3) * 2), ("band_hi", (u64 * 3) * 2), ("tail_first", u64 * 2)]


class BandOut(C.Structure):
    _fields_ = [("sum", (f64 * 3) * TML_SERIES_PER_STEP), ("cnt", (u64 * 3) * TML_SERIES_PER_STEP),
                ("tail_first", f64 * TML_SERIES_PER_STEP), ("tail_last", f64 * TML_SERIES_PER_STEP)]


class ProcAgg(C.Structure):
    _fields_ = [("n", u64), ("n_gpu", u64), ("ts_min", f64), ("ts_max", f64),
                ("sum_cpu", f64), ("max_cpu", f64), ("sum_rss", f64), ("max_rss", f64),
                ("sum_used", f64), ("max_used", f64), ("sum_resv", f64), ("max_resv", f64),
                ("max_total", f64), ("max_ratio", f64), ("max_cores", u32),
                ("any_gpu_available", u32), ("sum_cpu_lo", f64)]


class Comm(C.Structure):
    _fields_ = [("nccl_comm", vp), ("rank", i32), ("world", i32)]


XCHG = {"auto": 0, "p2p": 1, "a2a": 2}
XCHG_NAME = {0: "auto", 1: "p2p", 2: "a2a", 3: "local"}


class ReduceRunArgs(C.Structure):
    _fields_ = [("window", u32), ("proc_rows", u32), ("exchange", u32), ("speculate", u32)]


class KindResultC(C.Structure):
    _fields_ = [("observed", u32), ("n_used", u32), ("used", i32 * TML_MAX_RANKS),
                ("n_common", u64), ("start_step", u64), ("end_step", u64),
                ("n_rows", u64 * TML_MAX_RANKS), ("t_sums", (f64 * 7) * TML_MAX_RANKS),
                ("m_sums", (f64 * 4) * TML_MAX_RANKS), ("has_bands", u32), ("_pad", u32),
                ("band_sum", (f64 * 3) * 16), ("band_cnt", (u64 * 3) * 16),
                ("tail_first", f64 * 16), ("tail_last", f64 * 16),
                ("shard_lo", u64), ("shard_hi", u64), ("series", vp)]


class ReduceRunOut(C.Structure):
    _fields_ = [("n_ranks", u32), ("exchange_used", u32), ("fused_pass", u32), ("n_exchanges", u32),
                ("infos", WinInfo * TML_MAX_RANKS), ("procs", ProcAgg * TML_MAX_RANKS),
                ("time", KindResultC), ("mem", KindResultC), ("k3a_ms", f64), ("k4_ms", f64),
                ("stage_ms", f64 * 5)]


class SectionsArgs(C.Structure):
    _fields_ = [("ram_total", f64), ("gpu_count", i32), ("window", u32), ("proc_rows", u32), ("_pad", u32)]


class RankMeans(C.Structure):
    _fields_ = [("rank", i32), ("steps_analyzed", i64), ("dataloader_ms", f64), ("forward_ms", f64),
                ("backward_ms", f64), ("optimizer_ms", f64), ("step_cpu_ms", f64)]


class TrendIn(C.Structure):
    _fields_ = [("valid", i32), ("baseline_avg", f64), ("mid_avg", f64), ("recent_avg", f64)]


class StDiagIn(C.Structure):
    _fields_ = [("n_ranks", i32), ("max_rows", i32), ("n_common", i64), ("completed_step", i64),
                ("ranks", RankMeans * TML_MAX_RANKS), ("trend_step", TrendIn),
                ("trend_wait", TrendIn), ("trend_dl", TrendIn)]


class MemMetricIn(C.Structure):
    _fields_ = [("n_ranks", i32), ("ranks", i32 * TML_MAX_RANKS), ("rank_peak", f64 * TML_MAX_RANKS),
                ("trend_worst", TrendIn), ("trend_median", TrendIn), ("points", i32),
                ("tail_first", f64), ("tail_last", f64)]


class MemDiagIn(C.Structure):
    _fields_ = [("steps_used", i64), ("window_size", i32), ("completed_step", i64),
                ("ranks_seen", i32), ("gpu_total_bytes", f64), ("n_metrics", i32),
                ("metric", MemMetricIn * 2)]


class ProcDiagIn(C.Structure):
    _fields_ = [("n_ranks", i32), ("ranks", i32 * TML_MAX_RANKS), ("agg", ProcAgg * TML_MAX_RANKS),
                ("ram_total", f64 * TML_MAX_RANKS), ("gpu_count", i32 * TML_MAX_RANKS)]


assert C.sizeof(StepRecord) == 128 and C.sizeof(ProcRecord) == 64

# name -> (restype, argtypes); every symbol include/traceml_b200.h declares
SIGNATURES = {
    "tml_init": (C.c_int, [C.c_int, C.c_int, C.c_int, u32, u32, C.POINTER(vp)]),
    "tml_shutdown": (C.c_int, [vp]),
    "tml_abi_version": (u32, []),
    "tml_last_error": (C.c_char_p, []),
    "tml_status_str": (C.c_char_p, [C.c_int]),
    "tml_phase_begin": (C.c_int, [vp, u32, vp]),
    "tml_phase_end": (C.c_int, [vp, u32, C.c_int, vp]),
    "tml_phase_host": (C.c_int, [vp, u32, u64]),
    "tml_step_commit": (C.c_int, [vp, u64, u64, u64, u32, f64, vp]),
    "tml_step_discard": (C.c_int, [vp]),
    "tml_drain": (C.c_int, [vp, vp, u32, C.POINTER(u32), C.POINTER(u64)]),
    "tml_live": (C.c_int, [vp, C.POINTER(LiveStats)]),
    "tml_proc_commit": (C.c_int, [vp, C.POINTER(ProcRecord), vp]),
    "tml_proc_drain": (C.c_int, [vp, vp, u32, C.POINTER(u32), C.POINTER(u64)]),
    "tml_step_count": (u64, [vp]),
    "tml_proc_count": (u64, [vp]),
    "tml_launch_count": (u64, [vp]),
    "tml_ring_load": (C.c_int, [vp, vp, u64, vp]),
    "tml_proc_load": (C.c_int, [vp, vp, u64, vp]),
    "tml_ring_reset": (C.c_int, [vp]),
    "tml_win_prepare": (C.c_int, [vp, u32, vp, C.POINTER(WinInfo)]),
    "tml_win_presence": (C.c_int, [vp, u32, u64, u64, vp, vp]),
    "tml_win_select": (C.c_int, [vp, u32, u64, u64, vp, u32, vp, C.POINTER(AlignInfo)]),
    "tml_win_select_dense": (C.c_int, [vp, u32, u64, u64, vp, C.POINTER(AlignInfo)]),
    "tml_win_rows": (vp, [vp, u32]),
    "tml_win_rows_export": (C.c_int, [vp, u32, vp, C.POINTER(u64)]),
    "tml_peer_open": (C.c_int, [vp, vp, C.POINTER(vp)]),
    "tml_peer_close": (C.c_int, [vp, vp]),
    "tml_win_reduce": (C.c_int, [vp, C.POINTER(ReduceArgs), vp]),
    "tml_kernel_ms": (C.c_double, [vp, u32]),
    "tml_struct_size": (u64, [C.c_char_p]),
    "tml_sections_json": (C.c_int, [C.POINTER(ReduceRunOut), C.POINTER(SectionsArgs), vp, C.c_size_t]),
    "tml_win_set_defer": (C.c_int, [vp, C.c_int]),
    "tml_win_peek": (C.c_int, [vp, u32, C.POINTER(u64), C.POINTER(u64)]),
    "tml_win_fused": (C.c_int, [vp, u32, vp, vp, C.POINTER(WinInfo), C.POINTER(AlignInfo), C.POINTER(u32)]),
    "tml_win_exact_collect": (C.c_int, [vp, vp, C.POINTER(f64)]),
    "tml_win_exact_stats": (C.c_int, [vp, C.POINTER(u64)]),
    "tml_layer_init": (C.c_int, [vp, u32, u32]),
    "tml_layer_begin": (C.c_int, [vp, vp]),
    "tml_layer_end": (C.c_int, [vp, u32, u32, C.c_int, u64, vp]),
    "tml_layer_commit": (C.c_int, [vp, u64, vp]),
    "tml_layer_drain": (C.c_int, [vp, vp, u32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u64)]),
    "tml_xs_host_sum": (C.c_int, [vp, u64, C.c_int, C.POINTER(f64), C.POINTER(u64)]),
    "tml_reduce_run": (C.c_int, [vp, C.POINTER(Comm), C.POINTER(ReduceRunArgs), vp, C.POINTER(ReduceRunOut)]),
    "tml_combined_prepare": (C.c_int, [vp, u32, u32, vp, C.POINTER(CombinedInfo)]),
    "tml_combined_presence": (C.c_int, [vp, u32, u64, u64, vp, vp]),
    "tml_combined_select": (C.c_int, [vp, u32, u64, u64, vp, u32, vp, C.POINTER(CombinedAlign)]),
    "tml_combined_rows": (vp, [vp, u32]),
    "tml_combined_steps": (C.c_int, [vp, u32, C.POINTER(u64), u64, vp]),
    "tml_combined_series": (C.c_int, [vp, C.POINTER(vp), u32, u64, u32, u32, vp, vp]),
    "tml_win_bands": (C.c_int, [vp, vp, C.POINTER(BandArgs), vp, C.POINTER(BandOut)]),
    "tml_proc_reduce": (C.c_int, [vp, u32, vp, C.POINTER(ProcAgg)]),
    "tml_proc_reduce_launch": (C.c_int, [vp, u32, vp]),
    "tml_proc_reduce_collect": (C.c_int, [vp, C.POINTER(ProcAgg)]),
    "tml_diag_step_time": (C.c_int, [C.POINTER(StDiagIn), C.c_char_p, C.c_size_t]),
    "tml_diag_step_memory": (C.c_int, [C.POINTER(MemDiagIn), C.c_char_p, C.c_size_t]),
    "tml_diag_process": (C.c_int, [C.POINTER(ProcDiagIn), C.c_char_p, C.c_size_t]),
}

_LIB: Optional[C.CDLL] = None


class TraceMLNativeError(RuntimeError):
    """A libtraceml_b200 call returned a negative status."""


def lib() -> C.CDLL:
    """Load the native library once.  Raises if it is missing or stale."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"traceml_b200: native extension not found at {LIB_PATH}. Build it with "
            "`python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
            "There is no CPU fallback."
        )
    handle = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if the .so lacks a declared symbol
        fn.restype = restype
        fn.argtypes = argtypes
    ver = handle.tml_abi_version()
    if ver != 1:
        raise ImportError(f"traceml_b200: ABI version {ver} != 1 ({LIB_PATH} is stale)")
    _LIB = handle
    return handle


def check(status: int, what: str = "") -> int:
    if status < 0:
        l = lib()
        msg = (l.tml_last_error() or b"").decode("utf-8", "replace")
        name = (l.tml_status_str(status) or b"").decode()
        raise TraceMLNativeError(f"{what or 'libtraceml_b200'}: {name} ({status}) {msg}".strip())
    return status


_DIAG_BUF = None


def diag_json(fn_name: str, arg: C.Structure, cap: int = 1 << 16) -> Any:
    """Run one of the tml_diag_* engines and parse its JSON."""
    global _DIAG_BUF
    l = lib()
    if _DIAG_BUF is None or len(_DIAG_BUF) < cap:
        _DIAG_BUF = C.create_string_buffer(cap)
    buf = _DIAG_BUF
    rc = getattr(l, fn_name)(C.byref(arg), buf, len(buf))
    if rc == -8:  # TML_ERR_SMALL
        return diag_json(fn_name, arg, len(buf) * 8)
    check(rc, fn_name)
    return json.loads(buf.value)


_SEC_BUF = None


def sections_json(run_out, ram_total: float, gpu_count: int, window: int, proc_rows: int) -> Any:
    """tml_sections_json -> dict; rank-keyed step-time tables get their int keys back."""
    global _SEC_BUF
    if _SEC_BUF is None:
        _SEC_BUF = C.create_string_buffer(1 << 18)
    args = SectionsArgs(float(ram_total), int(gpu_count), int(window), int(proc_rows or 0), 0)
    rc = lib().tml_sections_json(C.byref(run_out), C.byref(args), _SEC_BUF, len(_SEC_BUF))
    if rc == -8:  # TML_ERR_SMALL
        _SEC_BUF = C.create_string_buffer(len(_SEC_BUF) * 8)
        return sections_json(run_out, ram_total, gpu_count, window, proc_rows)
    check(rc, "tml_sections_json")
    return Sections(_SEC_BUF.value)


class Sections:
    """The three sections of one reduce: a read-only mapping over the JSON text the native emitter
    produced.  The text is the product (it is what ``final_summary.json`` stores); the Python
    objects are a view of it, built on first access -- a summary that is only written to disk, or
    only asked for its diagnosis label, never pays for the rest.  ``reduce`` (the raw reduce
    output) and anything else the caller attaches live beside the parsed sections."""

    __slots__ = ("raw", "_parsed", "_extra")

    def __init__(self, raw: bytes):
        self.raw = raw
        self._parsed = None
        self._extra = {}

    def _get(self):
        if self._parsed is None:
            res = json.loads(self.raw)
            data = res["step_time"]["data"]
            for key in ("aligned_summary", "per_global_rank_summary"):  # rank-keyed tables: int keys back
                data[key] = {int(k): v for k, v in data[key].items()}
            self._parsed = res
        return self._parsed

    def __getitem__(self, key):
        if key in self._extra:
            return self._extra[key]
        return self._get()[key]

    def __setitem__(self, key, value):
        self._extra[key] = value

    def __contains__(self, key):
        return key in self._extra or key in self._get()

    def __iter__(self):
        yield from self._get()
        yield from self._extra

    def __len__(self):
        return len(self._get()) + len(self._extra)

    def get(self, key, default=None):
        return self[key] if key in self else default

    def keys(self):
        return list(self)

    def items(self):
        return [(k, self[k]) for k in self]

    def pop(self, key, *default):
        if key in self._extra:
            return self._extra.pop(key)
        return self._get().pop(key, *default)

    def to_dict(self):
        return dict(self.items())
