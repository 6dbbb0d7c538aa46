"""ctypes binding of ``libtraceml_b200.so`` (declared in ``include/traceml_b200.h``).

This is the only place Python crosses into native code.  Loading fails loudly:
there is no pure-Python or CPU fallback for any entry point.
"""

from __future__ import annotations

import ctypes as C
import json
import operator
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
TML_GRAPH_STEP_FAILED = 0x80000000  # tml_graph_step_commit: the step's body raised, keep the old id
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


class LayerSnap(C.Structure):
    _fields_ = [("cur_fwd_ns", u64), ("cur_bwd_ns", u64), ("peak_fwd_ns", u64), ("peak_bwd_ns", u64),
                ("flags", u32), ("last_fwd", u32), ("last_bwd", u32), ("_pad", u32)]


class LayerTickRow(C.Structure):
    _fields_ = [("cur_fwd_ms", f64), ("cur_bwd_ms", f64), ("peak_fwd_ms", f64), ("peak_bwd_ms", f64),
                ("worst_rank", i32), ("flags", u32), ("peak_last", u32 * 2), ("cur_rank", C.c_uint16 * 2),
                ("peak_rank", C.c_uint16 * 2)]


LAYER_HAS_FWD, LAYER_HAS_BWD = 1, 2
LSNAP_CUR_FWD, LSNAP_CUR_BWD, LSNAP_PEAK_FWD, LSNAP_PEAK_BWD = 1, 2, 4, 8
LSNAP_RANK_FWD, LSNAP_RANK_BWD = 16, 32


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
                ("sum_cpu", f64), ("max_cpu", f64), ("sum_rss", u64), ("max_rss", f64),
                ("sum_used", u64), ("max_used", f64), ("sum_resv", u64), ("max_resv", f64),
                ("max_total", f64), ("max_ratio", f64), ("max_cores", u32),
                ("any_gpu_available", u32), ("sum_cpu_lo", f64)]
    _BYTE_SUMS = frozenset(("sum_rss", "sum_used", "sum_resv"))

    def __setattr__(self, name, value):
        # The byte sums are exact u64 integers.  A caller may still hand one over as a float (they
        # were doubles before): it is taken as the nearest integer, exact for any integral value.
        if name in self._BYTE_SUMS and not isinstance(value, int):
            try:
                value = operator.index(value)  # numpy integers, without a detour through float
            except TypeError:
                value = int(round(float(value)))
        super().__setattr__(name, value)


TML_SYS_MAX_GPUS = 16
SYS_GPU_AVAILABLE = 1


class SysGpu(C.Structure):
    _fields_ = [("util", u32), ("temp_c", u32), ("mem_used", u64), ("mem_total", u64),
                ("power_mw", u32), ("power_limit_mw", u32)]


class SysRecord(C.Structure):
    _fields_ = [("seq", u64), ("ts", f64), ("cpu_pct", f64), ("ram_used", u64), ("ram_total", u64),
                ("flags", u32), ("gpu_count", u32), ("n_gpus", u32), ("_pad0", u32), ("_pad1", u64),
                ("gpu", SysGpu * TML_SYS_MAX_GPUS)]


class SysGpuAgg(C.Structure):
    _fields_ = [("n", u64), ("util_avg", f64), ("util_peak", f64), ("mem_avg", f64), ("mem_peak", f64),
                ("mem_total", f64), ("temp_avg", f64), ("temp_peak", f64), ("power_avg", f64),
                ("power_peak", f64), ("power_limit", f64)]


class SysAgg(C.Structure):
    _fields_ = [("n", u64), ("n_gpu", u64), ("first_ts", f64), ("last_ts", f64),
                ("cpu_avg", f64), ("cpu_peak", f64), ("ram_avg", f64), ("ram_peak", f64), ("ram_total", f64),
                ("gpu_util_avg", f64), ("gpu_util_peak", f64), ("gpu_mem_avg", f64), ("gpu_mem_peak", f64),
                ("gpu_temp_avg", f64), ("gpu_temp_peak", f64), ("gpu_power_avg", f64), ("gpu_power_peak", f64),
                ("gpu_available", u32), ("gpu_count", u32), ("n_gpus", u32), ("_pad", u32),
                ("gpu", SysGpuAgg * TML_SYS_MAX_GPUS)]


class SysDiagIn(C.Structure):
    _fields_ = [("node_rank", i32), ("_pad", i32), ("node_label", C.c_char * 32), ("agg", SysAgg)]


TML_HOSTNAME_MAX = 64


class SysPart(C.Structure):
    _fields_ = [("cpu_hi", f64), ("cpu_lo", f64), ("cpu_max", f64), ("ts_min", f64), ("ts_max", f64),
                ("d_hi", f64 * 4), ("d_lo", f64 * 4), ("d_max", f64 * 4),
                ("ram_sum", u64), ("ram_max", u64), ("ram_total_max", u64), ("n", u64), ("n_gpu", u64),
                ("avail", u32), ("gpu_count", u32), ("n_gpus", u32), ("_pad", u32)]


class SysNodeIdent(C.Structure):
    _fields_ = [("global_rank", i32), ("local_rank", i32), ("node_rank", i32), ("world_size", i32),
                ("local_world_size", i32), ("_pad", i32), ("hostname", C.c_char * TML_HOSTNAME_MAX)]


class SysNodeRecord(C.Structure):
    _fields_ = [("ident", SysNodeIdent), ("valid", u32), ("_pad", u32), ("agg", SysAgg), ("part", SysPart)]


class SysClusterOut(C.Structure):
    _fields_ = [("agg", SysAgg), ("n_nodes", u32), ("n_dup", u32), ("order", i32 * TML_MAX_RANKS)]


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
                ("m_sums", (f64 * 4) * TML_MAX_RANKS), ("has_bands", u32), ("series_paired", u32),
                ("band_sum", (f64 * 3) * 16), ("band_cnt", (u64 * 3) * 16),
                ("tail_first", f64 * 16), ("tail_last", f64 * 16),
                ("shard_lo", u64), ("shard_hi", u64), ("series", vp), ("series_ld", u64)]


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


assert C.sizeof(StepRecord) == 128 and C.sizeof(ProcRecord) == 64 and C.sizeof(SysRecord) == 576
assert C.sizeof(LayerSnap) == 48 and C.sizeof(LayerTickRow) == 56

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
    "tml_graph_phase_begin": (C.c_int, [vp, u32, vp]),
    "tml_graph_phase_end": (C.c_int, [vp, u32, C.c_int, vp]),
    "tml_graph_layer_begin": (C.c_int, [vp, vp]),
    "tml_graph_layer_end": (C.c_int, [vp, u32, u32, C.c_int, u64, vp]),
    "tml_graph_refs": (u64, []),
    "tml_graph_step_begin": (C.c_int, [vp, vp]),
    "tml_graph_step_commit": (C.c_int, [vp, u32, vp]),
    "tml_graph_step_publish": (C.c_int, [vp, u64, u64, u64, vp]),
    "tml_graph_step_id": (C.c_int, [vp, C.POINTER(u64)]),
    "tml_graph_phase_host": (C.c_int, [vp, u32, u64, vp]),
    "tml_graph_layer_commit": (C.c_int, [vp, vp]),
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
    "tml_layer_tick_bounds": (C.c_int, [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]),
    "tml_layer_tick_snapshot": (C.c_int, [vp, u64, vp, vp]),
    "tml_layer_tick_fold": (C.c_int, [vp, vp, u32, u32, vp, vp]),
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
    "tml_sys_commit": (C.c_int, [vp, C.POINTER(SysRecord), vp]),
    "tml_sys_load": (C.c_int, [vp, vp, u64, vp]),
    "tml_sys_count": (u64, [vp]),
    "tml_sys_read": (C.c_int, [vp, vp, u32, C.POINTER(u32), vp]),
    "tml_sys_reduce_launch": (C.c_int, [vp, u32, vp]),
    "tml_sys_reduce_collect": (C.c_int, [vp, C.POINTER(SysAgg)]),
    "tml_diag_system": (C.c_int, [C.POINTER(SysDiagIn), C.c_char_p, C.c_size_t]),
    "tml_sys_host_sum": (C.c_int, [vp, u64, u32, u32, C.POINTER(f64)]),
    "tml_sys_node_pack": (C.c_int, [vp, C.POINTER(SysNodeIdent), vp, vp]),
    "tml_sys_cluster_launch": (C.c_int, [vp, vp, u32, vp]),
    "tml_sys_cluster_collect": (C.c_int, [vp, vp]),
    "tml_diag_system_cluster": (C.c_int, [C.POINTER(SysDiagIn), u32, C.POINTER(SysAgg), C.c_char_p, C.c_size_t]),
    "tml_sys_host_cluster": (C.c_int, [C.POINTER(SysNodeRecord), u32, C.POINTER(SysClusterOut)]),
    # private (csrc/tml_internal.h): tml_reduce_run that emits an earlier reduce's sections meanwhile
    "tml_summary_run_": (C.c_int, [vp, C.POINTER(Comm), C.POINTER(ReduceRunArgs), vp, C.POINTER(ReduceRunOut),
                                   C.POINTER(ReduceRunOut), C.POINTER(SectionsArgs), vp, C.c_size_t,
                                   C.POINTER(C.c_int)]),
    # private: K6s on the native driver's side stream, behind the caller's stream
    "tml_sys_reduce_beside_": (C.c_int, [vp, u32, vp]),
    # private: the step ring's records rebuilt from its device layout; tml_ring_load's staging chunk
    "tml_ring_read_": (C.c_int, [vp, u64, u64, vp, vp]),
    "tml_ring_load_chunk_": (u64, []),
    # private: the dense-window certificate the ring's writers keep, for the last `window` rows
    "tml_ring_certified_": (C.c_int, [vp, u32]),
    # private: that certificate and every retained record within the ring's packed copy
    "tml_ring_packed_": (C.c_int, [vp, u32]),
    # private: the layer ring's contents replaced by host records (tests seed the layer tick with it)
    "tml_layer_load_": (C.c_int, [vp, vp, u64, vp]),
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


def diag_system_cluster(nodes, n_nodes: int, cluster: SysAgg) -> Any:
    """tml_diag_system_cluster over ``nodes`` (a ctypes array of SysDiagIn) -> dict."""
    global _DIAG_BUF
    cap = 1 << 16
    while True:
        if _DIAG_BUF is None or len(_DIAG_BUF) < cap:
            _DIAG_BUF = C.create_string_buffer(cap)
        rc = lib().tml_diag_system_cluster(nodes, int(n_nodes), C.byref(cluster), _DIAG_BUF, len(_DIAG_BUF))
        if rc != -8:  # TML_ERR_SMALL
            break
        cap = len(_DIAG_BUF) * 8
    check(rc, "tml_diag_system_cluster")
    return json.loads(_DIAG_BUF.value)


_SEC_BUF = None


def _sections_text(run_out, args) -> bytes:
    global _SEC_BUF
    if _SEC_BUF is None:
        _SEC_BUF = C.create_string_buffer(1 << 18)
    rc = lib().tml_sections_json(C.byref(run_out), C.byref(args), _SEC_BUF, len(_SEC_BUF))
    if rc == -8:  # TML_ERR_SMALL
        _SEC_BUF = C.create_string_buffer(len(_SEC_BUF) * 8)
        return _sections_text(run_out, args)
    check(rc, "tml_sections_json")
    # string_at: strlen + one copy; .value walks the 256 KB buffer byte by byte in Python's C loop
    return C.string_at(_SEC_BUF)


def sections_json(run_out, ram_total: float, gpu_count: int, window: int, proc_rows: int) -> Any:
    """tml_sections_json -> dict; rank-keyed step-time tables get their int keys back."""
    args = SectionsArgs(float(ram_total), int(gpu_count), int(window), int(proc_rows or 0), 0)
    return Sections(_sections_text(run_out, args))


_PREV_BUF = None


def summary_run(handle, comm, run_args, run_out, stream: int, prev: "Sections") -> None:
    """tml_reduce_run into ``run_out``; while its pass runs, the native driver emits the text of
    ``prev`` (the sections of an earlier reduce, from their own copy of its result), which it
    would otherwise emit on first access."""
    global _PREV_BUF
    if _PREV_BUF is None:
        _PREV_BUF = C.create_string_buffer(1 << 18)
    prc = C.c_int(0)
    check(lib().tml_summary_run_(handle, C.byref(comm), C.byref(run_args), stream, C.byref(run_out),
                                 C.byref(prev._src), C.byref(prev._args), _PREV_BUF, len(_PREV_BUF), C.byref(prc)),
          "tml_summary_run_")
    if prc.value == 0 and prev._raw is None:
        prev._raw = C.string_at(_PREV_BUF)
    # else (TML_ERR_SMALL, ...): prev emits its text itself on first access, and reports errors there


class Sections:
    """The three sections of one reduce: a read-only mapping over the JSON text the native emitter
    produced.  The text is the product (it is what ``final_summary.json`` stores); the Python
    objects are a view of it, built on first access -- a summary that is only written to disk, or
    only asked for its diagnosis label, never pays for the rest.  ``reduce`` (the raw reduce
    output) and anything else the caller attaches live beside the parsed sections."""

    __slots__ = ("_raw", "_src", "_args", "_parsed", "_extra")

    def __init__(self, raw: Optional[bytes] = None, src=None, args=None):
        """``raw``: the text; or ``src`` (a ReduceRunOut the object owns) and ``args`` (SectionsArgs)
        to emit it from, on first access unless ``summary_run`` has emitted it before."""
        self._raw = raw
        self._src, self._args = src, args
        self._parsed = None
        self._extra = {}

    @property
    def raw(self) -> bytes:
        if self._raw is None:
            self._raw = _sections_text(self._src, self._args)
        return self._raw

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

    def __reduce__(self):
        """Pickles as the text, the parsed sections if there are any (the caller may have changed
        them) and what the caller attached.  The emitter's input stays behind: it has a pointer
        field, which ctypes cannot pickle, and is not needed once the text exists."""
        return (_sections_restore, (self.raw, self._parsed, self._extra))


def _sections_restore(raw, parsed, extra) -> Sections:
    s = Sections(raw)
    s._parsed, s._extra = parsed, extra
    return s
