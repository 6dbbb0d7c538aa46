"""GPU: the step ring's 32-B packed records and the window pass's packed stream.

``k_commit``, ``k_commit_dev`` and ``k_ring_split`` store a packed copy of each record's durations
and peaks (five 36-bit and two 38-bit fields) and raise ``wide_mark`` for a record that does not fit
it; the single-rank window pass streams the packed copies of a certified window whose retained
records all fit.  For every case below:

* ``tml_ring_packed_`` equals a numpy restatement on the records the ring retains: certified, and
  every retained row's five summarised durations below 2^36 and both peaks below 2^38;
* the certificate, the window pass called directly and the build's sections check as in
  ``test_gpu_dense_certificate.py`` (counters, series bit for bit against ``fast_oracle.series16``,
  row-level oracles; above the bulk threshold the chained build against the staged one);
* two rings holding the same window, one with a wide row before t_start (so one streams packed
  records and the other hot halves), give byte-identical section JSON, series, band sums and tails.

Cases: each field at 2^k - 1 (fits) and 2^k (wide), through a load and through commits; every field at
its largest fitting value; a wide row at the oldest retained row, at a tile edge, at the ring seam, on
a staging-chunk edge, just before t_start and just scrolled out; a load, host commits, a load then
commits, commits then a load, a load with more records than slots; commits from a captured graph and
host commits in device-committed mode; reset, then reuse.
"""
import functools

import numpy as np
import pytest
import torch

import series_geometry as sg
import test_gpu_dense_certificate as dc
from test_gpu_graph_steps import _capture_steps, _eager_steps, _graph_model, fresh  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

DUR_BITS, MEM_BITS = 36, 38
FIELDS = {"dl": 0, "fwd": 2, "bwd": 3, "opt": 4, "wall": 5, "peak_alloc": None, "peak_resv": None}


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _recs(n, seed, first_step=1000):
    """series_geometry's dense records brought inside the packed ranges (no duration becomes 0)."""
    r = sg.step_records(n, seed, first_step=first_step)
    d = r["dur_ns"]
    r["dur_ns"] = np.where(d >> np.uint64(DUR_BITS), d >> np.uint64(6), d)
    r["peak_alloc"] = r["peak_alloc"] >> np.uint64(3)
    r["peak_resv"] = r["peak_resv"] >> np.uint64(3)
    return r


def _set(recs, rows, field, value):
    out = recs.copy()
    for r in rows:
        col = FIELDS[field]
        if col is None:
            out[field][r] = np.uint64(value)
        else:
            d = out["dur_ns"][r]
            d[col] = np.uint64(value)
            out["dur_ns"][r] = d
    return out


def _wide(recs, rows):
    return _set(recs, rows, "dl", 1 << DUR_BITS)


def _packed_restated(recs, W):
    fits = (recs["dur_ns"][:, sg.USABLE_COLS] < np.uint64(1 << DUR_BITS)).all() and \
        (recs["peak_alloc"] < np.uint64(1 << MEM_BITS)).all() and (recs["peak_resv"] < np.uint64(1 << MEM_BITS)).all()
    return dc._restated(recs, W) and bool(fits)


def _check(eng, slots, W, want=None):
    """The packed verdict against its restatement, then everything test_gpu_dense_certificate checks."""
    from traceml_b200 import _abi

    recs = dc._retained(eng, slots)
    verdict = _abi.lib().tml_ring_packed_(eng.handle, int(W))
    assert verdict == int(_packed_restated(recs, W))
    if want is not None:
        assert verdict == int(want)
    dc._check(eng, slots, W)
    return verdict


def _run(slots, W, ops, want):
    eng = dc._engine(slots)
    try:
        dc._apply(eng, ops)
        _check(eng, slots, W, want)
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 1. field edges
EDGES = [(f, k) for f in FIELDS for k in ("fits", "wide")]


@pytest.mark.parametrize("writer", ["load", "commit"])
@pytest.mark.parametrize("field,kind", EDGES)
def test_field_edge(cuda, writer, field, kind):
    bits = DUR_BITS if FIELDS[field] is not None else MEM_BITS
    value = (1 << bits) - 1 if kind == "fits" else 1 << bits
    if writer == "load":   # window rows 1096.. of 4096: the edge row is inside the window
        slots, W, recs, row = 4096, 3000, _recs(4096, 50), 2000
    else:
        slots, W, recs, row = 64, 40, _recs(100, 51), 80
    _run(slots, W, [(writer, _set(recs, [row], field, value))], kind == "fits")


@pytest.mark.parametrize("writer", ["load", "commit"])
def test_every_field_at_its_largest(cuda, writer):
    slots, W, n = (4096, 3000, 4096) if writer == "load" else (64, 40, 100)
    recs = _recs(n, 52)
    for f in FIELDS:
        bits = DUR_BITS if FIELDS[f] is not None else MEM_BITS
        recs = _set(recs, [n - 7, n - 3], f, (1 << bits) - 1)
    _run(slots, W, [(writer, recs)], True)


# ----------------------------------------------------------------------------- 2. where the wide row sits
@functools.lru_cache(maxsize=None)
def _cases():
    ch = dc._chunk()
    big = 2 * ch + 100
    d = _recs
    return {
        # name: (slots, window, ops, packed)
        "commits_only": (64, 50, [("commit", d(200, 1))], True),
        "load_only": (big + 100, 200_000, [("load", d(big, 2))], True),
        "load_then_commits": (4096, 3000, [("load", d(3000, 3)), ("commit", d(200, 4, first_step=1000 + 3000))], True),
        "commits_then_load": (4096, 3000, [("commit", d(150, 5)), ("load", d(3000, 6, first_step=1000 + 150))], True),
        # the wide record is among those the load drops: the ring never holds it
        "load_more_than_slots": (4113, 3001, [("load", _wide(d(10_000, 7), [100]))], True),
        "wide_oldest": (4096, 3000, [("load", _wide(d(4096, 8), [0]))], False),
        "wide_tile_edge_31": (4096, 3000, [("load", _wide(d(4096, 9), [31]))], False),
        "wide_tile_edge_32": (4096, 3000, [("load", _wide(d(4096, 10), [32]))], False),
        # slots 1025 after 1500 records: the seam (slot 0) at retained row 550
        "wide_seam": (1025, 1000, [("load", _wide(d(1500, 11), [1025]))], False),
        "wide_chunk_edge": (big + 100, 200_000, [("load", _wide(d(big, 12), [ch]))], False),
        # window 3000 of 4096 rows: t_start = 1096
        "wide_before_t_start": (4096, 3000, [("load", _wide(d(4096, 13), [1095]))], False),
        "wide_commit_before_t_start": (64, 40, [("commit", _wide(d(100, 14), [59]))], False),
        # the wide record leaves the ring: packed again
        "wide_scrolled_out_commit": (64, 40, [("commit", _wide(d(100, 15), [35]))], True),
        "wide_scrolled_out_load": (4096, 3000, [("load", _wide(d(4096, 16), [10])),
                                                ("commit", d(20, 17, first_step=1000 + 4096))], True),
        # not certified: never packed
        "gap": (4096, 4000, [("load", dc._with(d(4096, 18), [1000], step=5))], False),
    }


CASE_NAMES = ["commits_only", "load_only", "load_then_commits", "commits_then_load", "load_more_than_slots",
              "wide_oldest", "wide_tile_edge_31", "wide_tile_edge_32", "wide_seam", "wide_chunk_edge",
              "wide_before_t_start", "wide_commit_before_t_start", "wide_scrolled_out_commit",
              "wide_scrolled_out_load", "gap"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_packed_verdict(cuda, name):
    slots, W, ops, want = _cases()[name]
    _run(slots, W, ops, want)


def test_reset_then_reuse(cuda):
    slots, W = 4096, 3000
    eng = dc._engine(slots)
    try:
        dc._apply(eng, [("load", _wide(_recs(4096, 40), [3500]))])
        assert _check(eng, slots, W, False) == 0
        eng.reset()
        dc._apply(eng, [("load", _recs(4096, 41, first_step=7))])   # wide_mark starts over
        assert _check(eng, slots, W, True) == 1
        dc._apply(eng, [("commit", _recs(10, 42, first_step=7 + 4096))])
        assert _check(eng, slots, W, True) == 1
        eng.reset()
        dc._apply(eng, [("commit", _wide(_recs(10, 43, first_step=3), [4]))])
        assert _check(eng, slots, W, False) == 0
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 3. packed vs hot halves
@pytest.mark.parametrize("n,W", [(140_000, 135_000), (4096, 3000)])
def test_packed_and_hot_streams_agree(cuda, n, W):
    """The same window with and without a wide row before t_start: the two rings take the two
    certified streams and every output is the same bytes."""
    import replay
    from traceml_b200 import _abi, sections

    recs = _recs(n, 60)
    outs = []
    for want, ring in ((1, recs), (0, _wide(recs, [n - W - 1]))):
        eng = dc._engine(n)
        try:
            eng.load_steps(ring)
            torch.cuda.synchronize()
            assert _abi.lib().tml_ring_certified_(eng.handle, W) == 1
            assert _abi.lib().tml_ring_packed_(eng.handle, W) == want
            rc, info, ok, ser = dc._fused(eng, W, W)
            assert rc == 0 and ok == 1
            got = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, W)
            red = got["reduce"]
            assert bool(red.fused_rows) == (W > dc.BULK)
            k = [ser.tobytes(), got.raw]
            for part in (red.time, red.mem):
                k.append(part.series.cpu().numpy().tobytes())
                k += [np.array(x, dtype=np.float64).tobytes()
                      for x in (part.band_sum, part.band_cnt, list(part.tail_first), list(part.tail_last))]
            outs.append(k)
        finally:
            eng.close()
    assert outs[0] == outs[1]


# ----------------------------------------------------------------------------- 4. device-committed mode
def test_captured_commits(fresh):
    """k_commit_dev: commits replayed from a captured graph fit; a host commit in device-committed
    mode with a wide duration breaks the packed verdict while the ring retains it."""
    import traceml_b200 as traceml
    from helpers import build_vs_row_oracles
    from traceml_b200 import _abi

    eng = fresh
    lib = _abi.lib()
    model, opt, x, y = _graph_model()
    _eager_steps(traceml, model, opt, x, y, 2)
    g, _ = _capture_steps(traceml, model, opt, x, y, 2)
    for _ in range(4):
        g.replay()
    torch.cuda.synchronize()
    n = eng.step_count
    assert n == 10
    recs = dc._retained(eng, n)
    assert len(recs) == n and list(recs["step"]) == list(range(1, n + 1))
    for w in (1, 4, n):
        assert lib.tml_ring_packed_(eng.handle, w) == int(_packed_restated(recs, w)) == 1
    # a host commit through k_commit_dev with a wide data-loader time
    s = torch.cuda.current_stream().cuda_stream
    assert eng.phase_host(0, 1 << DUR_BITS) == 0
    assert eng.phase_host(2, 1000) == 0
    assert eng.step_commit(n + 1, 4096, 8192, sg.FLAG_HAS_MEM, 0.0, s) == 0
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    recs = dc._retained(eng, n + 5)
    assert len(recs) == n + 5 and int(recs["dur_ns"][n, 0]) == 1 << DUR_BITS
    for w in (1, 4, n + 5):
        assert lib.tml_ring_certified_(eng.handle, w) == 1
        assert lib.tml_ring_packed_(eng.handle, w) == int(_packed_restated(recs, w)) == 0
    build_vs_row_oracles(eng, recs, len(recs))
    build_vs_row_oracles(eng, recs, 4)
    del g
