"""GPU: the dense-window certificate kept by the step ring's writers.

``k_commit`` and ``k_ring_split`` raise three marks (a step-id gap, a record without memory, an
unusable record) as records land; the single-rank window pass streams a certified window without
re-checking its density.  For every case below:

* the certificate (``tml_ring_certified_``) equals a numpy restatement of what the host's density
  check accepts, on the records the ring retains: (a) consecutive step ids after the first retained
  row, (b) memory on every retained row, (c) every row from t_start on usable;
* the window pass called directly accepts exactly the certified windows, with the counters of its
  numpy restatement and the per-step series bit for bit (``fast_oracle.series16``);
* the build's sections equal the row-level oracles, and above the bulk threshold the chained
  build's series equal the Python-sequenced staged build's.

Cases: commits only; a load only; a load then commits; commits then a load; a load with more
records than slots; ring wraps; a gap on a staging-chunk edge, at the window's first row (allowed)
and at its second; a duplicated and a decreasing step id; a row without memory at the oldest row,
at a tile edge and at the ring seam; an unusable row just before t_start and at it; reset, then reuse.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import series_geometry as sg
from helpers import build_vs_row_oracles

pytestmark = pytest.mark.gpu

BULK = 1 << 17   # the native build's single-rank bulk threshold (TML_FUSED_MIN_ROWS)


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _chunk():
    from traceml_b200 import _abi

    return int(_abi.lib().tml_ring_load_chunk_())


def _recs(n, seed, first_step=1000):
    return sg.step_records(n, seed, first_step=first_step)


def _commit(eng, recs):
    """Each record through the step path: host phase durations, then one commit."""
    s = torch.cuda.current_stream().cuda_stream
    for r in recs:
        for p in range(6):
            if int(r["dur_ns"][p]):
                eng.phase_host(p, int(r["dur_ns"][p]))
        assert eng.step_commit(int(r["step"]), int(r["peak_alloc"]), int(r["peak_resv"]), int(r["flags"]),
                               0.0, s) == 0


def _apply(eng, ops):
    for kind, recs in ops:
        if kind == "load":
            eng.load_steps(recs)
        else:
            _commit(eng, recs)
        torch.cuda.synchronize()


def _retained(eng, slots):
    from traceml_b200 import _abi
    from traceml_b200.records import STEP_RECORD_DTYPE

    total = eng.step_count
    n = min(total, slots)
    out = torch.empty(n * 128, dtype=torch.uint8, device="cuda")
    _abi.check(_abi.lib().tml_ring_read_(eng.handle, total - n, n, out.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream), "tml_ring_read_")
    torch.cuda.synchronize()
    return out.cpu().numpy().view(STEP_RECORD_DTYPE).copy()


def _restated(recs, W):
    """(a)-(c) on the retained records (oldest first)."""
    step = recs["step"].astype(np.uint64)
    t0 = max(0, len(recs) - W)
    a = bool((step[1:] == step[:-1] + np.uint64(1)).all())
    b = bool(((recs["flags"] & np.uint32(sg.FLAG_HAS_MEM)) != 0).all())
    c = bool((recs["dur_ns"][t0:, sg.USABLE_COLS] > 0).any(axis=1).all())
    return a and b and c


def _fused(eng, W, n_win):
    from traceml_b200 import _abi

    buf = torch.zeros(16 * n_win, dtype=torch.float64, device="cuda")
    info, al, ok = _abi.WinInfo(), _abi.AlignInfo(), C.c_uint32(7)
    rc = _abi.lib().tml_win_fused(eng.handle, int(W), buf.data_ptr(), 0, C.byref(info), C.byref(al), C.byref(ok))
    torch.cuda.synchronize()
    return rc, info, int(ok.value), buf.cpu().numpy().reshape(16, n_win)


def _check(eng, slots, W, want=None):
    """Everything the module docstring lists, for eng's ring with window W; returns the verdict."""
    import replay
    from oracle import fast_oracle
    from traceml_b200 import _abi, sections

    recs = _retained(eng, slots)
    verdict = _abi.lib().tml_ring_certified_(eng.handle, int(W))
    assert verdict == int(_restated(recs, W))
    if want is not None:
        assert verdict == int(want)
    n_win = min(W, len(recs))
    rc, info, ok, ser = _fused(eng, W, n_win)
    step = recs["step"].astype(np.int64)
    if (np.diff(step) < 0).any():
        assert rc == _abi.TML_ERR_NONMONOTONIC and ok == 0
        with pytest.raises(_abi.TraceMLNativeError, match=r"step ids decrease"):
            sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, W)
        return verdict
    assert rc == 0, _abi.lib().tml_last_error()
    assert ok == verdict
    c = sg.window_counters(recs, W, rule="fused")
    assert [int(info.n_cand[0]), int(info.n_cand[1]), int(info.t_count), int(info.n_both), int(info.dup_rows)] == \
        [c["n_cand"][0], c["n_cand"][1], c["t_count"], c["n_both"], c["dup_rows"]]
    assert list(info.dense) == c["dense"] and list(info.lo) == c["lo"] and list(info.hi) == c["hi"]
    exp = fast_oracle.series16(fast_oracle.window_rows(recs[len(recs) - n_win:])[None])
    assert ser.tobytes() == exp.tobytes()
    got = build_vs_row_oracles(eng, recs, W)
    red = got["reduce"]
    assert bool(red.fused_rows) == (bool(verdict) and n_win > BULK)
    if n_win > BULK:
        chained = (red.time.series.cpu().numpy().copy(), red.mem.series.cpu().numpy().copy())
        staged = sections.SummaryEngine([eng], native=False, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                        gpu_count=1).build(W, W)["reduce"]
        assert staged.time.series.cpu().numpy().tobytes() == chained[0].tobytes()
        assert staged.mem.series.cpu().numpy().tobytes() == chained[1].tobytes()
    if verdict:
        t_rows = fast_oracle.window_rows(recs[len(recs) - n_win:])
        s16 = fast_oracle.series16(t_rows[None])
        assert red.time.series.cpu().numpy()[:12].tobytes() == s16[:12].tobytes()
    return verdict


def _engine(slots):
    from traceml_b200.engine import Engine

    return Engine(device=0, rank=0, world=1, ring_slots=slots, proc_slots=64)


def _with(recs, rows, *, step=None, nomem=False, unusable=False):
    out = recs.copy()
    for r in rows:
        if step is not None:
            # shift this row and every later one: one break at r
            out["step"][r:] = (out["step"][r:].astype(np.int64) + step).astype(np.uint64)
        if nomem:
            out["flags"][r] = 0
        if unusable:
            d = out["dur_ns"][r]
            d[:] = 0
            d[1] = 7   # only h2d > 0
            out["dur_ns"][r] = d
    return out


@functools.lru_cache(maxsize=None)
def _cases():
    ch = _chunk()
    big = 2 * ch + 100
    d = _recs
    return {
        # name: (slots, window, ops, certified)
        "commits_only": (64, 50, [("commit", d(200, 1))], True),
        "load_only": (big + 100, 200_000, [("load", d(big, 2))], True),
        "load_then_commits": (4096, 3000, [("load", d(3000, 3)), ("commit", d(200, 4, first_step=1000 + 3000))], True),
        "commits_then_load": (4096, 3000, [("commit", d(150, 5)), ("load", d(3000, 6, first_step=1000 + 150))], True),
        "load_more_than_slots": (4113, 3001, [("load", d(10_000, 7))], True),
        "ring_wraps": (1025, 1000, [("load", d(700, 8)), ("commit", d(40, 9, first_step=1700)),
                                    ("load", d(700, 10, first_step=1740)), ("load", d(700, 11, first_step=2440))], True),
        # a gap on the edge of staging chunk 1: the step id before it comes from the caller's buffer
        "gap_chunk_edge": (big + 100, 200_000, [("load", d(10, 12)), ("load", _with(d(big, 13), [ch], step=5))], False),
        # the ring keeps exactly the second chunk: the gap sits on its first row (allowed), or its second
        "gap_first_row": (ch, ch, [("load", d(10, 14)), ("load", _with(d(2 * ch, 15), [ch], step=5))], True),
        "gap_second_row": (ch, ch, [("load", d(10, 16)), ("load", _with(d(2 * ch, 17), [ch + 1], step=5))], False),
        "gap_first_row_commit": (64, 64, [("commit", _with(d(128, 18), [64], step=3))], True),
        "gap_second_row_commit": (64, 64, [("commit", _with(d(128, 19), [65], step=3))], False),
        "duplicate": (4096, 4000, [("load", _with(d(4096, 20), [1000], step=-1))], False),
        "decreasing": (4096, 4000, [("load", _with(d(4096, 21), [1000], step=-2))], False),
        "decreasing_commit": (64, 64, [("commit", _with(d(100, 22), [70], step=-2))], False),
        "nomem_oldest": (4096, 3000, [("load", _with(d(4096, 23), [0], nomem=True))], False),
        "nomem_tile_edge": (4096, 3000, [("load", _with(d(4096, 24), [31], nomem=True))], False),
        "nomem_commit": (64, 40, [("commit", _with(d(100, 25), [60], nomem=True))], False),
        "nomem_evicted": (64, 40, [("commit", _with(d(100, 26), [35], nomem=True))], True),
        # slots 1025 after 1500 records: the seam (slot 0) at retained row 550
        "nomem_seam": (1025, 1000, [("load", _with(d(1500, 27), [1025], nomem=True))], False),
        # window 3000 of 4096 rows: t_start = 1096
        "unusable_before_t_start": (4096, 3000, [("load", _with(d(4096, 28), [1095], unusable=True))], True),
        "unusable_at_t_start": (4096, 3000, [("load", _with(d(4096, 29), [1096], unusable=True))], False),
        "unusable_commit_before_t_start": (64, 40, [("commit", _with(d(100, 30), [59], unusable=True))], True),
        "unusable_commit_at_t_start": (64, 40, [("commit", _with(d(100, 31), [60], unusable=True))], False),
    }


CASE_NAMES = ["commits_only", "load_only", "load_then_commits", "commits_then_load", "load_more_than_slots",
              "ring_wraps", "gap_chunk_edge", "gap_first_row", "gap_second_row", "gap_first_row_commit",
              "gap_second_row_commit", "duplicate", "decreasing", "decreasing_commit", "nomem_oldest",
              "nomem_tile_edge", "nomem_commit", "nomem_evicted", "nomem_seam", "unusable_before_t_start",
              "unusable_at_t_start", "unusable_commit_before_t_start", "unusable_commit_at_t_start"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_certificate(cuda, name):
    slots, W, ops, want = _cases()[name]
    eng = _engine(slots)
    try:
        _apply(eng, ops)
        _check(eng, slots, W, want)
    finally:
        eng.close()


def test_reset_then_reuse(cuda):
    slots, W = 4096, 3000
    eng = _engine(slots)
    try:
        _apply(eng, [("load", _with(_recs(4096, 40), [2000], nomem=True))])
        assert _check(eng, slots, W, False) == 0
        eng.reset()
        _apply(eng, [("load", _recs(4096, 41, first_step=7))])   # the marks and the last step id start over
        assert _check(eng, slots, W, True) == 1
        _apply(eng, [("commit", _recs(10, 42, first_step=7 + 4096))])
        assert _check(eng, slots, W, True) == 1
        eng.reset()
        _apply(eng, [("commit", _recs(10, 43, first_step=3))])   # no predecessor after a reset
        assert _check(eng, slots, W, True) == 1
    finally:
        eng.close()
