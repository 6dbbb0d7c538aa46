"""GPU: the alignment stages (K3b presence, K3c select, K3d gather) and the trend bands (K4b),
each called on its own through the engine and compared with a numpy restatement written here.

* K3b: presence bytes for each kind's candidate flags, with ``glo`` below, at and above the rank's
  first step, at spans on every 16-byte word edge and 4096-byte block edge, and at a span above
  4 194 304 step ids with fewer than 100 rows.  Re-flushed step ids (the ``duplicates`` replay) keep
  at most one candidate row per step id and kind -- the precondition of K3b's unsynchronised
  ``rowof`` stores.
* K3c: the selected steps and rows, exactly, at every ``count16`` edge, at 1, 2, 1024, 1025 and
  about 1300 count blocks (one and two trips of the single-block scan), with the last block partly
  filled, an empty presence map, one set byte at either end, and ``W`` = 1, total - 1, total, total + 1.
  The bytes past ``span`` in the presence buffer are ones, so a count that reads past the span
  shows.
* K3d: the aligned rows byte for byte, through the copy path and the contiguous path on the same
  rows, with a row-index break at j = 1 and at j = nsel - 1; the byte sums exactly (totals above
  2^53), the maxima exactly, the time sums in the reference's order (K3e) and the memory kind's float
  sums within the bound of the gather's tree depth.  ``win_select_dense`` gives what ``win_select``
  gives on a dense window.
* K4b: counts, tails and band sums bit for bit at shard edges before, at, inside and past each
  band: a band held whole by the shard is summed as the reference's mean sums it (CPython's
  compensated ``sum()``, left to right); a
  band split across shards in the kernel's tree order (thread t sums the indices t mod 256 in
  order, then ``block_sum``).  Per-shard results add up to the whole series.
* Both drivers' band layouts (``tml_reduce_run``'s C++ ``trend_layout`` and the Python-sequenced
  ``SummaryEngine._bands``): band counts, tails and sums of one-rank builds against the oracle's
  band bounds over the build's own series; the single-rank bulk build (its (16, 5) ``k_bands``
  launch over a series whose row stride exceeds its length) against ``tml_win_bands``.
* The trend gates: seeded series whose step-time trend is exactly +8 % in real arithmetic, where
  a tree-ordered band mean lands one ulp under the gate and the reference's mean on it (seed 29: a
  plain left-to-right sum lands under it too), through one-rank staged and bulk builds and a two-rank build: the whole step-time diagnosis
  (note text included) and the step-memory diagnosis equal the oracle's.
"""
import math

import numpy as np
import pytest
import torch

from helpers import assert_struct, plain, strip_device
from test_trend_layout_cpu import _oracle_layout

pytestmark = pytest.mark.gpu

KIND_TIME, KIND_MEM = 0, 1
SEL_TILE = 4096
U = 2.0 ** -53  # unit roundoff of f64
BIG = 1 << 50   # peak_alloc base: a few rows already sum above 2^53
ID0 = 1 << 40   # peak_resv = ID0 + row identity: tells the aligned rows apart


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


# ----------------------------------------------------------------------------- inputs
def _records(steps, seed):
    """One rank's StepRecords with these step ids; peak_resv carries each row's identity."""
    from traceml_b200.records import (FLAG_HAS_MEM, PHASE_BACKWARD, PHASE_DATALOADER, PHASE_FORWARD,
                                      PHASE_OPTIMIZER, PHASE_STEP, STEP_RECORD_DTYPE)

    rng = np.random.default_rng(seed)
    steps = np.asarray(steps, dtype=np.uint64)
    n = len(steps)
    rec = np.zeros(n, dtype=STEP_RECORD_DTYPE)
    rec["step"] = steps
    for p, lo, hi in ((PHASE_DATALOADER, 1_000_000, 9_000_000), (PHASE_FORWARD, 5_000_000, 15_000_000),
                      (PHASE_BACKWARD, 10_000_000, 30_000_000), (PHASE_OPTIMIZER, 1_000_000, 5_000_000),
                      (PHASE_STEP, 20_000_000, 60_000_000)):
        rec["dur_ns"][:, p] = rng.integers(lo, hi, n).astype(np.uint64)
    rec["n_calls"][:] = 1
    rec["peak_alloc"] = (BIG + rng.integers(0, 1 << 30, n)).astype(np.uint64)
    rec["peak_resv"] = (ID0 + np.arange(n)).astype(np.uint64)
    rec["host_ts"] = 1.7e9 + np.arange(n) * 0.04
    rec["gpu_mask"] = 0b11100
    rec["flags"] = FLAG_HAS_MEM
    rec["seq"] = np.arange(n, dtype=np.uint64)
    return rec


def _junk(step):
    """A record that is a candidate of neither kind: no phase time, no memory."""
    from traceml_b200.records import STEP_RECORD_DTYPE

    r = np.zeros(1, dtype=STEP_RECORD_DTYPE)
    r["step"] = step
    return r


def _sparse_steps(span, k, seed, first=1000):
    """k sorted step ids in [first, first + span), the first and the last of them included."""
    rng = np.random.default_rng(seed)
    mid = rng.choice(np.arange(1, span - 1), size=k - 2, replace=False)
    return first + np.sort(np.concatenate([[0, span - 1], mid]))


def _engine(recs):
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=len(recs) + 8, proc_slots=64)
    if len(recs):
        eng.load_steps(recs)
    torch.cuda.synchronize()
    return eng


# ----------------------------------------------------------------------------- numpy restatements
def _cands(recs):
    """The window pass's candidate flags over a window holding every record (k_window_rows):
    time -- the oldest usable row of its run of equal step ids; memory -- a row with memory that is
    the last of its run or followed by a row without memory."""
    from traceml_b200.records import FLAG_HAS_MEM, PHASE_BACKWARD, PHASE_DATALOADER, PHASE_FORWARD, \
        PHASE_OPTIMIZER, PHASE_STEP

    n = len(recs)
    st = recs["step"].astype(np.int64)
    d = recs["dur_ns"]
    usable = (d[:, [PHASE_DATALOADER, PHASE_FORWARD, PHASE_BACKWARD, PHASE_OPTIMIZER, PHASE_STEP]] > 0).any(axis=1)
    has_mem = (recs["flags"] & FLAG_HAS_MEM) != 0
    cand_t = np.zeros(n, bool)
    seen = set()
    for i in range(n):
        if i == 0 or st[i] != st[i - 1]:
            seen = set()
        if usable[i] and not seen:
            cand_t[i] = True
        if usable[i]:
            seen.add(i)
    nxt_diff = np.ones(n, bool)
    nxt_diff[:-1] = (st[1:] != st[:-1]) | ~has_mem[1:]
    cand_m = has_mem & nxt_diff
    return cand_t, cand_m


def _expected_presence(recs, kind, glo, span):
    cand = _cands(recs)[kind]
    st = recs["step"].astype(np.int64)[cand]
    out = np.zeros(span, np.uint8)
    keep = (st >= glo) & (st < glo + span)
    out[st[keep] - glo] = 1
    return out


def _padded(span):
    return (span + 15) // 16 * 16 + 16


def _presence(eng, kind, glo, span):
    """K3b into a buffer whose bytes past ``span`` are ones (K3b must leave them alone)."""
    buf = torch.ones(_padded(span), dtype=torch.uint8, device="cuda")
    eng.win_presence(kind, glo, span, buf)
    torch.cuda.synchronize()
    return buf


def _depth_bound(values, depth):
    """First-order bound of any summation tree in which no value passes through more than ``depth``
    additions: depth * u * sum |x|."""
    return depth * U * math.fsum(abs(float(x)) for x in values)


def _check_aligned(eng, recs, kind, glo, span, pres, W):
    """K3c + K3d over presence bytes ``pres`` (a subset of this rank's own presence, as after the
    cross-rank MIN), against numpy: steps, rows, sums."""
    from oracle import fast_oracle as fo

    buf = _presence(eng, kind, glo, span)
    buf[:span] = torch.from_numpy(pres).to("cuda")
    a = eng.win_select(kind, glo, span, buf, W)
    idx = np.flatnonzero(pres)
    total = idx.size
    keep = min(total, W)
    assert a.n_common == keep, (a.n_common, keep)
    if keep == 0:
        assert eng.win_rows_ptr(kind) == 0
        return a
    sel_steps = glo + idx[total - keep:]
    assert (a.start_step, a.end_step, a.n_rows) == (int(sel_steps[0]), int(sel_steps[-1]), keep)
    cand = _cands(recs)[kind]
    rowof = {int(s): i for i, s in enumerate(recs["step"]) if cand[i]}
    sel_rows = np.array([rowof[int(s)] for s in sel_steps])
    rows = fo.window_rows(recs)
    x = rows[sel_rows]
    got = eng.win_rows_tensor(kind, keep).view(keep, 8).cpu().numpy()
    assert got.tobytes() == x.tobytes()
    # byte sums exact, maxima exact
    m_exp = [float(int(recs["peak_alloc"][sel_rows].astype(object).sum())),
             float(int(recs["peak_resv"][sel_rows].astype(object).sum())), x[:, 6].max(), x[:, 7].max()]
    assert list(a.m_sums) == m_exp
    d = fo.derived(x)
    traced = d["step_time"]
    elems = [d["dataloader_fetch"], d["forward"], d["backward"], d["optimizer_step"], np.maximum(0.0, traced),
             traced, d["dataloader_fetch"] + traced]
    if kind == KIND_TIME:  # K3e: the reference's order, newest first
        assert list(a.t_sums) == [fo.seq_sum(e[::-1]) for e in elems]
    else:
        # k_gather: a thread chain of at most ceil(4 keep / 256) trips, 3 shuffle levels, 8 warps,
        # then k_finalize (lane chains of ceil(grid / 32) <= ceil(4 keep / 8192) blocks, 5 levels)
        depth = -(-4 * keep // 256) + 3 + 8 + -(-4 * keep // 8192) + 5
        for k, e in enumerate(elems):
            assert abs(a.t_sums[k] - math.fsum(e)) <= _depth_bound(e, depth), k
    return a


# ----------------------------------------------------------------------------- K3b presence
@pytest.mark.parametrize("span", [1, 15, 16, 17, 4095, 4096, 4097])
@pytest.mark.parametrize("shift", [-3, 0, 2])
def test_presence_word_and_tile_edges(cuda, span, shift):
    steps = np.arange(100, 100 + 5000, dtype=np.int64)
    steps = np.delete(steps, [1, 5, 16, 17, 300, 4094, 4095])  # holes at word and tile edges
    recs = _records(steps, seed=span)
    eng = _engine(recs)
    try:
        eng.win_prepare(10_000)
        glo = 100 + shift
        for kind in (KIND_TIME, KIND_MEM):
            buf = _presence(eng, kind, glo, span).cpu().numpy()
            assert buf[:span].tobytes() == _expected_presence(recs, kind, glo, span).tobytes(), kind
            assert (buf[span:] == 1).all(), "K3b wrote past the span"
    finally:
        eng.close()


def test_presence_wide_sparse_span(cuda):
    span = 4_194_304 + 1_000_003
    recs = _records(_sparse_steps(span, 90, seed=1), seed=1)
    eng = _engine(recs)
    try:
        eng.win_prepare(10_000)
        for kind in (KIND_TIME, KIND_MEM):
            buf = _presence(eng, kind, 1000, span).cpu().numpy()
            assert buf[:span].tobytes() == _expected_presence(recs, kind, 1000, span).tobytes()
            assert int(buf[:span].sum()) == 90
    finally:
        eng.close()


def test_duplicates_keep_one_candidate_per_step(cuda):
    """A re-flushed step id is two adjacent rows of one id: one time candidate (the older) and one
    memory candidate (the newer) per id, and the aligned rows are exactly those."""
    import replay

    recs = replay.make_step_replay("duplicates", 1, 300, seed=4)[0]
    recs["peak_resv"] = ID0 + np.arange(len(recs), dtype=np.uint64)
    assert len(recs) == 302
    eng = _engine(recs)
    try:
        info = eng.win_prepare(10_000)
        for kind in (KIND_TIME, KIND_MEM):
            cand = _cands(recs)[kind]
            st = recs["step"][cand]
            assert np.unique(st).size == st.size == 300  # the precondition, in the restatement
            assert info.n_cand[kind] == 300               # ... and in the device's own flags
            glo, span = int(info.lo[kind]), int(info.hi[kind] - info.lo[kind] + 1)
            pres = _presence(eng, kind, glo, span).cpu().numpy()[:span]
            _check_aligned(eng, recs, kind, glo, span, pres, 10_000)
    finally:
        eng.close()


# ----------------------------------------------------------------------------- K3c select, K3d gather
# (span, rows): 1, 2, 1024, 1025 and ~1300 count blocks; the last block full or partly filled
WIDE = [(SEL_TILE, 40), (SEL_TILE + 1, 40), (1024 * SEL_TILE, 60), (1024 * SEL_TILE + 1, 60),
        (1300 * SEL_TILE - 777, 90)]


@pytest.mark.parametrize("span,k", WIDE)
def test_select_blocks_and_scan_trips(cuda, span, k):
    recs = _records(_sparse_steps(span, k, seed=span), seed=span)
    eng = _engine(recs)
    try:
        eng.win_prepare(10_000)
        for kind in (KIND_TIME, KIND_MEM):
            pres = _presence(eng, kind, 1000, span).cpu().numpy()[:span]
            for W in (1, k - 1, k, k + 1):
                _check_aligned(eng, recs, kind, 1000, span, pres, W)
        # a set byte only at either end, and none
        for only in (0, span - 1):
            one = np.zeros(span, np.uint8)
            one[only] = 1
            a = _check_aligned(eng, recs, KIND_TIME, 1000, span, one, 5)
            assert a.start_step == a.end_step == 1000 + only
        _check_aligned(eng, recs, KIND_TIME, 1000, span, np.zeros(span, np.uint8), 5)
    finally:
        eng.close()


@pytest.mark.parametrize("span", [1, 15, 16, 17, 31, 33, 4095, 4096, 4097])
def test_select_word_edges(cuda, span):
    """Dense and gapped presence over spans at the 16-byte word edges of count16."""
    steps = np.arange(500, 500 + span + 40, dtype=np.int64)
    steps = np.delete(steps, [2, 14, 15][: max(0, min(3, span - 2))])
    recs = _records(steps, seed=span + 7)
    eng = _engine(recs)
    try:
        eng.win_prepare(10_000)
        for kind in (KIND_TIME, KIND_MEM):
            pres = _presence(eng, kind, 500, span).cpu().numpy()[:span]
            total = int(pres.sum())
            for W in sorted({1, max(1, total - 1), max(1, total), total + 1}):
                _check_aligned(eng, recs, kind, 500, span, pres, W)
    finally:
        eng.close()


@pytest.mark.parametrize("where", ["j1", "last"])
def test_gather_copy_and_contiguous_paths(cuda, where):
    """The same selected rows once contiguous (aligned rows = a slice of the window rows) and once
    with a non-candidate row inside them at j = 1 or j = nsel - 1 (the copy path)."""
    k = 300
    base = _records(np.arange(2, 2 * k + 2, 2), seed=9)  # even step ids 2 .. 2k
    at = 1 if where == "j1" else k - 1
    broken = np.concatenate([base[:at], _junk(int(base["step"][at]) - 1), base[at:]])
    outs = []
    for recs in (base, broken):
        eng = _engine(recs)
        try:
            eng.win_prepare(10_000)
            for kind in (KIND_TIME, KIND_MEM):
                span = 2 * k - 1
                pres = _presence(eng, kind, 2, span).cpu().numpy()[:span]
                assert int(pres.sum()) == k
                a = _check_aligned(eng, recs, kind, 2, span, pres, k)
                rows = eng.win_rows_tensor(kind, k).view(k, 8).cpu().numpy().tobytes()
                outs.append((kind, bytes(a), rows))
        finally:
            eng.close()
    assert outs[:2] == outs[2:]


@pytest.mark.parametrize("n,W", [(700, 700), (700, 256), (5000, 4097)])
def test_select_dense_matches_select(cuda, n, W):
    recs = _records(np.arange(7, 7 + n), seed=n + W)
    eng = _engine(recs)
    try:
        info = eng.win_prepare(10_000)
        for kind in (KIND_TIME, KIND_MEM):
            assert info.dense[kind] == 1
            lo, hi = int(info.lo[kind]), int(info.hi[kind])
            span = hi - lo + 1
            dense = eng.win_select_dense(kind, hi - W + 1, W)
            d_rows = eng.win_rows_tensor(kind, W).view(W, 8).cpu().numpy().tobytes()
            pres = _presence(eng, kind, lo, span).cpu().numpy()[:span]
            sel = _check_aligned(eng, recs, kind, lo, span, pres, W)
            s_rows = eng.win_rows_tensor(kind, W).view(W, 8).cpu().numpy().tobytes()
            assert bytes(dense) == bytes(sel), kind
            assert d_rows == s_rows
    finally:
        eng.close()


# ----------------------------------------------------------------------------- K4b bands
def bands_order_sum(v):
    """k_bands' order over the values v of a band split across shards (its part on one shard): thread t adds v[t], v[t + 256], ... in
    turn from 0.0; each warp folds its lanes with the xor butterfly 16, 8, 4, 2, 1; thread 0 adds the
    8 warp results in warp order from 0.0."""
    v = np.asarray(v, dtype=np.float64)
    pad = np.zeros(-(-v.size // 256) * 256)
    pad[: v.size] = v
    acc = np.zeros(256)
    for row in pad.reshape(-1, 256):
        acc = acc + row
    lanes = np.arange(32)
    x = 0.0
    for w in range(8):
        y = acc[w * 32:(w + 1) * 32].copy()
        for m in (16, 8, 4, 2, 1):
            y = y + y[lanes ^ m]
        x = x + y[0]
    return x


def _band_args(n, lay_t, lay_m, shard, tails):
    from traceml_b200 import _abi

    a = _abi.BandArgs()
    a.n_common, (a.shard_lo, a.shard_hi) = n, shard
    for k, lay in enumerate((lay_t, lay_m)):
        for b in range(3):
            a.band_lo[k][b], a.band_hi[k][b] = lay[b]
    a.tail_first[0], a.tail_first[1] = tails
    return a


def reference_sum(v):
    """The reference's band sum (core.py:34, CPython >= 3.12 ``sum()``): Neumaier's compensated sum,
    left to right from 0, the compensation added once at the end when it is finite and non-zero."""
    f = c = 0.0
    for x in np.asarray(v, dtype=np.float64).tolist():
        t = f + x
        c += (f - t) + x if abs(f) >= abs(x) else (x - t) + f
        f = t
    return f + c if c and math.isfinite(c) else f


def _expected_bands(series, n, lay_t, lay_m, shard, tails):
    lo_s, hi_s = shard
    sums, cnts, tf, tl = np.zeros((16, 3)), np.zeros((16, 3), np.int64), np.full(16, np.nan), np.full(16, np.nan)
    for s in range(16):
        kind = 1 if s >= 12 else 0
        lay = (lay_t, lay_m)[kind]
        for b in range(3):
            lo, hi = max(lay[b][0], lo_s), min(lay[b][1], hi_s)
            cnts[s, b] = max(0, hi - lo)
            if lay[b][0] < lay[b][1] and (lo, hi) == tuple(lay[b]):  # the whole band: the reference's sum
                sums[s, b] = reference_sum(series[s, lo:hi])
            else:
                sums[s, b] = bands_order_sum(series[s, lo:hi]) if hi > lo else 0.0
        f, last = tails[kind], n - 1
        if n and lo_s <= f < hi_s:
            tf[s] = series[s, f]
        if n and lo_s <= last < hi_s:
            tl[s] = series[s, last]
    return sums, cnts, tf, tl


def _run_bands(eng, dev_series, n, lay_t, lay_m, shard, tails):
    out = eng.win_bands(dev_series, _band_args(n, lay_t, lay_m, shard, tails))
    return (np.array([list(r) for r in out.sum]), np.array([list(r) for r in out.cnt], np.int64),
            np.array(list(out.tail_first)), np.array(list(out.tail_last)))


def _bits(x):
    return np.asarray(x, dtype=np.float64).tobytes()


# n not a multiple of 256; bands of 1, 255, 256, 257 and ~1000 points
BAND_CASES = [
    (1_000, [(100, 101), (300, 555), (900, 1000)], [(0, 256), (256, 513), (513, 1000)], (0, 999)),
    (3_333, [(333, 1334), (1500, 1755), (2900, 3333)], [(7, 8), (1000, 2001), (3000, 3333)], (2500, 17)),
]


@pytest.mark.parametrize("case", range(len(BAND_CASES)))
def test_bands_bits_and_shards(cuda, case):
    n, lay_t, lay_m, tails = BAND_CASES[case]
    rng = np.random.default_rng(case)
    series = rng.lognormal(0.0, 2.0, (16, n))  # magnitudes over decades: order shows in the last bits
    dev = torch.from_numpy(series).to("cuda")
    eng = _engine(_records([1], seed=0))
    try:
        edges = sorted({0, n} | {e for lay in (lay_t, lay_m) for b in lay for e in
                                 (b[0] - 1, b[0], b[0] + 1, (b[0] + b[1]) // 2, b[1] - 1, b[1], b[1] + 1)
                                 if 0 <= e <= n})
        whole = _run_bands(eng, dev, n, lay_t, lay_m, (0, n), tails)
        exp = _expected_bands(series, n, lay_t, lay_m, (0, n), tails)
        assert (whole[1] == exp[1]).all()
        for g, e in zip(whole[::2] + whole[3:], exp[::2] + exp[3:]):
            assert _bits(g) == _bits(e)
        # shards ending and starting at every edge, and some between two edges: each bit-exact
        shards = [(0, e) for e in edges] + [(e, n) for e in edges] + \
            [(a, b) for a in edges for b in edges if a <= b][::11]
        for lo, hi in shards:
            got = _run_bands(eng, dev, n, lay_t, lay_m, (lo, hi), tails)
            exp = _expected_bands(series, n, lay_t, lay_m, (lo, hi), tails)
            assert (got[1] == exp[1]).all(), (lo, hi)
            for g, e in ((got[0], exp[0]), (got[2], exp[2]), (got[3], exp[3])):
                assert _bits(g) == _bits(e), (lo, hi)
        cuts = [0] + edges[1:-1:3] + [n]
        parts = [_run_bands(eng, dev, n, lay_t, lay_m, (a, b), tails) for a, b in zip(cuts, cuts[1:])]
        assert (sum(p[1] for p in parts) == whole[1]).all()
        folded = np.zeros((16, 3))
        for p in parts:  # rank order, as bands_collect folds the shards
            folded = folded + p[0]
        for s in range(16):
            lay = (lay_t, lay_m)[1 if s >= 12 else 0]
            for b in range(3):
                v = series[s, lay[b][0]:lay[b][1]]
                # both sides against the exact sum: the whole band's compensated sum is within
                # 2u|sum| + O(n u^2) sum|x| (depth 3 covers both terms); a value of the folded side passes through its thread's chain
                # (ceil(size / 256)), the 5 butterfly levels, the 8 warp adds and the shard fold
                depth = 3 + (-(-v.size // 256) + 5 + 8 + len(parts))
                assert abs(folded[s, b] - whole[0][s, b]) <= _depth_bound(v, depth)
        for k in (2, 3):  # each tail comes from exactly one shard
            got = np.array([next((p[k][s] for p in parts if not np.isnan(p[k][s])), np.nan) for s in range(16)])
            assert _bits(got) == _bits(whole[k])
    finally:
        eng.close()


def test_bands_empty_series(cuda):
    dev = torch.zeros(16, dtype=torch.float64, device="cuda")
    eng = _engine(_records([1], seed=0))
    try:
        z = [(0, 0)] * 3
        s, c, tf, tl = _run_bands(eng, dev, 0, z, z, (0, 0), (0, 0))
        assert not s.any() and not c.any() and np.isnan(tf).all() and np.isnan(tl).all()
        # a shard that misses every band: counts 0, sums 0
        dev = torch.ones(16 * 600, dtype=torch.float64, device="cuda")
        s, c, tf, tl = _run_bands(eng, dev, 600, [(10, 20)] * 3, [(30, 40)] * 3, (100, 200), (0, 599))
        assert _bits(s) == _bits(np.zeros((16, 3))) and not c.any()
        assert np.isnan(tf).all() and np.isnan(tl).all()
    finally:
        eng.close()


# ----------------------------------------------------------------------------- layouts of both drivers
@pytest.mark.parametrize("n", [199, 200, 222, 223, 1_001, 10_001, 11_111])
@pytest.mark.parametrize("native", [True, False], ids=["native", "python"])
def test_build_band_layout(cuda, n, native):
    """A one-rank build's band counts, tails and sums over its own series, against the oracle's band
    bounds: the C++ trend_layout (tml_reduce_run) and the Python one (the sequenced reduce)."""
    import replay
    from traceml_b200 import sections

    recs = replay.make_step_replay("trend_worsening", 1, n, seed=n)[0]
    eng = _engine(recs)
    try:
        red = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1) \
            .build(n, n, timings=not native)["reduce"]
        k = red.time
        series = k.series.cpu().numpy().astype(np.float64)
        assert series.shape == (16, n)
        lay_t, lay_m = _oracle_layout(n, 200, 0.10), _oracle_layout(n, 50, 0.0)
        z = [(0, 0)] * 3
        exp = _expected_bands(series, n, lay_t or z, lay_m or z, (0, n), (0, n - min(n, 1000)))
        assert [[int(c) for c in r] for r in k.band_cnt] == exp[1].tolist()
        assert _bits([[float(x) for x in r] for r in k.band_sum]) == _bits(exp[0])
        assert _bits(list(k.tail_first)) == _bits(exp[2]) and _bits(list(k.tail_last)) == _bits(exp[3])
    finally:
        eng.close()


def test_bulk_build_bands_match_win_bands(cuda):
    """The single-rank bulk build (window above 2^17 rows): its chained (16, 5) k_bands launch reads
    the series at a row stride above its length; the band bits equal tml_win_bands over a plain
    copy of the same series, and the reference's sums of the oracle's bands."""
    import replay
    from traceml_b200 import sections

    n = (1 << 17) + 1_000
    recs = replay.make_step_replay("trend_worsening", 1, n, seed=5)[0]
    eng = _engine(recs)
    try:
        red = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(n, n)["reduce"]
        assert red.fused_rows
        k = red.time
        assert k.series.shape == (16, n) and k.series.stride(0) > n
        series = k.series.cpu().numpy()
        lay_t, lay_m = _oracle_layout(n, 200, 0.10), _oracle_layout(n, 50, 0.0)
        tails = (0, n - 1000)
        plain_out = _run_bands(eng, torch.from_numpy(np.ascontiguousarray(series)).to("cuda"), n, lay_t, lay_m,
                               (0, n), tails)
        exp = _expected_bands(series, n, lay_t, lay_m, (0, n), tails)
        got = (np.array([[float(x) for x in r] for r in k.band_sum]),
               np.array([[int(c) for c in r] for r in k.band_cnt], np.int64),
               np.array(list(k.tail_first)), np.array(list(k.tail_last)))
        for g, p, e in zip(got, plain_out, exp):
            assert g.tobytes() == p.tobytes() and _bits(g) == _bits(e)
    finally:
        eng.close()


# ----------------------------------------------------------------------------- the trend gates
# Seeds whose baseline band (25 ms + offsets of a few ns that cancel, in a seeded order) has a
# mean in the reference's summation that puts pct = (27 - base) / base at exactly 0.08, while a tree order
# gives 0.07999999999999985: the reference prints "worsening (↑ +8.0%)", a tree-summed band none.
GATE_SEEDS = (12, 29)


def _gate_records(n, seed, first=1):
    """Step time = backward only (exact ns / 10^6 ms): 26 ms, with 25 ms +- cancelling offsets over
    the baseline band and 27 ms over the recent band of the oracle's layout."""
    from traceml_b200.records import FLAG_HAS_MEM, PHASE_BACKWARD, STEP_RECORD_DTYPE

    (b0, b1), _, (r0, r1) = _oracle_layout(n, 200, 0.10)
    ns = np.full(n, 26_000_000, np.int64)
    rng = np.random.default_rng(seed)
    k = b1 - b0
    d = rng.integers(1, 50, k // 2)
    off = np.concatenate([d, -d, np.zeros(k - 2 * (k // 2), np.int64)])
    rng.shuffle(off)
    ns[b0:b1] = 25_000_000 + off
    ns[r0:r1] = 27_000_000
    rec = np.zeros(n, dtype=STEP_RECORD_DTYPE)
    rec["step"] = np.arange(first, first + n)
    rec["dur_ns"][:, PHASE_BACKWARD] = ns
    rec["n_calls"][:] = 1
    rec["peak_alloc"] = 4 << 30
    rec["peak_resv"] = (4 << 30) + (256 << 20)
    rec["gpu_mask"] = 0b11100
    rec["flags"] = FLAG_HAS_MEM
    rec["host_ts"] = 1.7e9 + np.arange(n) * 0.03
    rec["seq"] = np.arange(n)
    return rec


def test_gate_seeds_split_the_orders():
    """The committed seeds are gate cases: the reference's order and the tree order disagree."""
    from oracle import trend_oracle

    for n in (12_000, (1 << 17) + 2_000):
        (b0, b1), _, (r0, r1) = _oracle_layout(n, 200, 0.10)
        for seed in GATE_SEEDS:
            v = _gate_records(n, seed)["dur_ns"][:, 3] / 1.0e6
            ref = trend_oracle._mean(v[b0:b1].tolist())
            assert ref == reference_sum(v[b0:b1]) / (b1 - b0)
            tree = bands_order_sum(v[b0:b1]) / (b1 - b0)
            assert (27.0 - ref) / ref == 0.08 and (27.0 - tree) / tree < 0.08


@pytest.mark.parametrize("seed", GATE_SEEDS)
@pytest.mark.parametrize("ranks,n", [(1, 12_000), (1, (1 << 17) + 2_000), (2, 12_000)],
                         ids=["one_rank", "one_rank_bulk", "two_ranks"])
def test_trend_gate_matches_oracle(cuda, seed, ranks, n):
    import replay
    from oracle import fast_oracle as fo
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    recs = {r: _gate_records(n, seed) for r in range(ranks)}
    engines = []
    for r in range(ranks):
        e = Engine(device=0, rank=r, world=ranks, ring_slots=n + 8, proc_slots=64)
        e.load_steps(recs[r])
        engines.append(e)
    torch.cuda.synchronize()
    try:
        got = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=ranks).build(n, n)
        if ranks == 1:
            assert got["reduce"].fused_rows == (n > (1 << 17))
        o = fo.step_time_section(recs, max_rows=n)
        assert o["diagnosis"]["primary"]["note"] == "Trend: step time is worsening (↑ +8.0%)."
        assert_struct(plain(got["step_time"]["diagnosis"]), plain(o["diagnosis"]), "diagnosis")
        mo = fo.step_memory_section(recs, window_size=n, gpu_total_bytes=got["step_memory"]["gpu_total_bytes"])
        gd, od = strip_device(plain(got["step_memory"]["diagnosis"])), strip_device(plain(mo["diagnosis"]))
        assert_struct(gd["primary"], od["primary"], "mem.primary")
        assert_struct(gd["issues"], od["issues"], "mem.issues")
    finally:
        for e in engines:
            e.close()
