"""GPU: K3e's reference-order window sums (csrc/tml_exact_sum.cuh) bit for bit, on the inputs its
machinery exists for.

The replay data K3e sees elsewhere is benign: 3-40 ms per phase, no running sum stalled near a
binade boundary, no exact round-half-even tie.  Here the records are adversarial -- a chain stalled
just below a power of two (every chunk unsafe: the tile-slot table and the walk's staging lists
overflow), exact ties on every add, giants that jump several binades inside one 32-row tile, whole
zero chunks, start-up crossings at every power of two -- and all windows but one (the 1024 side of
the switch) are large enough for the planned walk: more than 1024 summation positions, the leading
``pad`` included.

Everything is compared with ``==`` against ``oracle/fast_oracle.py`` (itself pinned ``==`` to the
row-level oracle and so to the reference): the per-rank window sums (``win_prepare``), the aligned
sums of each aligned row source (``win_select_dense`` / ``win_select``), the deferred side-stream
job, the aligned memory sums above 2^53 (including an exact halfway case) and the K4 per-step
series of the same windows.  The one exception is the world-of-one window of 2^17 + 1 rows, which
takes the documented tree sums (rel 1e-9).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import plain

pytestmark = pytest.mark.gpu

NS_MAX = (1 << 53) - 1            # every duration stays below 2^53 ns (ns -> ms proven exact-rounded there)
TIE_NS = 15_625                   # 1/64 ms: multiples of it convert to ms exactly
STALL_NS = int(round(2.0 ** 33 * (1.0 - 3.0e-7) * 1.0e6))  # 2^33 (1 - 3e-7) ms
TARGETS = (0, 2, 3, 4, 5)         # dl, fwd, bwd, opt, wall: the phases a family is applied to
FAMILIES = ("stall", "ties", "giant", "sparse", "startup", "lognormal", "mem")
XS_SLOT_CAP = 4096                # tml_exact_sum.cuh: (chunk, chain) pairs that may carry tile maps
GB = 10 ** 9


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------------ records
def make_records(family, n, target, seed, first_step=1):
    """``n`` StepRecords with unique increasing step ids and integer-ns durations < 2^53.

    ``family`` shapes the phase ``target`` (the others get the family's background values); odd
    rows have wall > compute, even rows wall < compute, unless the family drives the wall itself.
    The newest row is summed first (reference order), so "the newest row" is where a chain starts."""
    from traceml_b200.records import FLAG_HAS_MEM, STEP_RECORD_DTYPE

    rng = np.random.default_rng([seed, target, FAMILIES.index(family), n])
    q = 1
    if family == "stall":          # newest row: the chain just below 2^33 ms, then +1..2 ns per row
        d = rng.integers(1, 3, (n, 6))
        d[-1, target] = STALL_NS
    elif family == "ties":         # multiples of 1/64 ms, the target near 2^53 ns: past ~2^47 ms
        q = TIE_NS                 # running sum, a large share of the adds are exact ties
        d = rng.integers(0, 1 << 20, (n, 6)) * q
        d[:, target] = rng.integers((1 << 52) // q, NS_MAX // q, n) * q
    elif family == "giant":        # 1-3 ms rows; three giants, each jumping several binades
        d = rng.integers(1_000_000, 3_000_000, (n, 6))
        for j, g in enumerate((3 * 10 ** 12, 2 * 10 ** 15, 89 * 10 ** 14)):
            pos = (j + 1) * n // 5 // 256 * 256 + 141   # rows before it in summation order
            if pos < n:
                d[n - 1 - pos, target] = g
    elif family == "sparse":       # half the rows unusable (all zero, mostly whole chunks), opt 0
        d = np.exp(rng.normal(np.log(2.0e7), 0.7, (n, 6))).astype(np.int64) + 1
        d[:, 4] = 0
    elif family == "startup":      # 1-3 ns: a binade crossing at every power of two of the row count
        d = rng.integers(1, 4, (n, 6))
    elif family == "lognormal":    # catch-all: ~12 decades
        d = np.clip(np.exp(rng.normal(np.log(1.0e6), 5.0, (n, 6))), 1, 10 ** 15).astype(np.int64)
    elif family == "mem":          # ordinary durations; the peaks below are the point
        d = rng.integers(1_000_000, 40_000_000, (n, 6))
    else:
        raise ValueError(family)
    d = d.astype(np.int64)
    if target != 5:
        comp = d[:, 2] + d[:, 3] + d[:, 4]
        odd = (np.arange(n) & 1) == 1
        d[:, 5] = np.minimum(np.where(odd, comp + d[:, 5], comp // (2 * q) * q), NS_MAX // q * q)
    if family == "sparse":
        dead = np.repeat(rng.random((n + 511) // 512) < 0.5, 512)[:n] | (rng.random(n) < 0.05)
        d[dead] = 0
    assert d.min() >= 0 and d.max() <= NS_MAX
    rec = np.zeros(n, dtype=STEP_RECORD_DTYPE)
    rec["step"] = np.arange(first_step, first_step + n, dtype=np.uint64)
    rec["dur_ns"] = d.astype(np.uint64)
    rec["n_calls"] = 1
    if family == "mem":            # 80-180 GB peaks: the byte sums of >= 10^5 rows exceed 2^53
        alloc = rng.integers(80 * GB, 180 * GB, n)
        rec["peak_alloc"] = alloc.astype(np.uint64)
        rec["peak_resv"] = (alloc + rng.integers(0, 1 << 30, n)).astype(np.uint64)
    else:
        rec["peak_alloc"] = ((4 << 30) + rng.integers(0, 1 << 20, n)).astype(np.uint64)
        rec["peak_resv"] = rec["peak_alloc"] + np.uint64(256 << 20)
    rec["flags"] = FLAG_HAS_MEM
    rec["seq"] = np.arange(n, dtype=np.uint64)
    return rec


def target_of(rank, salt):
    return TARGETS[(rank + salt) % len(TARGETS)]


# ------------------------------------------------------------------------------------ engines
def _engines(records, ring=None, world=None):
    from traceml_b200.engine import Engine

    R = len(records)
    out = []
    for r in range(R):
        e = Engine(device=0, rank=r, world=world or R, ring_slots=ring or (len(records[r]) + 8), proc_slots=64)
        e.load_steps(records[r])
        out.append(e)
    torch.cuda.synchronize()
    return out


def _close(engines):
    for e in engines:
        e.close()


def _slow_rows(engine):
    """Rows the last K3e walk of this context added one by one, per chain."""
    from traceml_b200 import _abi

    buf = (C.c_uint64 * 7)()
    _abi.check(_abi.lib().tml_win_exact_stats(engine.handle, buf), "tml_win_exact_stats")
    return [int(v) for v in buf]


def _align(engines, infos, kind, W):
    """Stages 2-3 in one process: the lock-step shortcut when every window is dense, else the
    presence maps, their intersection (element-wise min) and ``win_select``."""
    part = [i for i, inf in enumerate(infos) if inf.n_cand[kind] > 0]
    glo = max(int(infos[i].lo[kind]) for i in part)
    ghi = min(int(infos[i].hi[kind]) for i in part)
    assert ghi >= glo
    span = ghi - glo + 1
    if all(infos[i].dense[kind] for i in part):
        n = min(span, W)
        return [e.win_select_dense(kind, ghi - n + 1, n) for e in engines]
    pres = None
    for e in engines:
        p = torch.empty(span, dtype=torch.uint8, device="cuda")
        e.win_presence(kind, glo, span, p)
        pres = p if pres is None else torch.minimum(pres, p)
    return [e.win_select(kind, glo, span, pres, W) for e in engines]


def _window_chains(kept, W):
    """The seven window-mode addends of one rank in summation order (newest first), zeros for the
    rows the section does not use -- what K3e adds position by position."""
    from oracle import fast_oracle

    d = fast_oracle.derived(fast_oracle.window_rows(kept[-W:]))
    usable = (d["dataloader_fetch"] > 0) | (d["forward"] > 0) | (d["backward"] > 0) | \
             (d["optimizer_step"] > 0) | (d["_cpu"] > 0)
    cols = [d["dataloader_fetch"], d["forward"], d["backward"], d["optimizer_step"], d["_cpu"], d["step_time"],
            d["dataloader_fetch"] + d["step_time"]]
    return [np.where(usable, c, 0.0)[::-1] for c in cols]


def _band_pairs(chains, pad, margin=0.5e-6):
    """(chunk, chain) pairs whose running sum lies inside the plan's margin band around a binade
    boundary, from the exact sequential prefix sums.  The plan (xs_plan) widens [lo, hi] by 1e-6
    relative; half of that here, so K3a's approximate chunk sums (relative error << 1e-7) can only
    make the device count larger.  Chunks with lo == 0 (start-up) never get a slot and are not
    counted."""
    total = 0
    for x in chains:
        z = np.concatenate([np.zeros(pad), x])
        pre = np.add.accumulate(z)
        nch = (len(z) + 255) // 256
        hi = pre[np.minimum(np.arange(1, nch + 1) * 256, len(z)) - 1]
        lo = np.concatenate([[0.0], hi[:-1]])
        band = (lo > 0) & (np.frexp(lo * (1 - margin))[1] != np.frexp(hi * (1 + margin))[1])
        total += int(band.sum())
    return total


def _oracle_aligned(kept, W):
    from oracle import fast_oracle

    parts = [fast_oracle.rank_part(k, W) for k in kept]
    common = fast_oracle.common_suffix([p["steps"] for p in parts], W)
    return parts, common, [fast_oracle.aligned_part(p, common) for p in parts]


def _exact_mem(rec, steps):
    pos = np.searchsorted(rec["step"].astype(np.int64), steps)
    a, r = rec["peak_alloc"][pos], rec["peak_resv"][pos]
    return [float(int(a.sum(dtype=np.uint64))), float(int(r.sum(dtype=np.uint64))), float(a.max()), float(r.max())]


def _check_aligned_time(engines, infos, kept, W, series=True):
    """Aligned time kind: sums, memory sums over the same rows and (optionally) K4's series."""
    from oracle import fast_oracle
    from traceml_b200 import _abi

    _, common, al = _oracle_aligned(kept, W)
    got = _align(engines, infos, _abi.KIND_TIME, W)
    n = int(common.size)
    for r, a in enumerate(got):
        assert int(a.n_common) == n and int(a.start_step) == int(common[0]) and int(a.end_step) == int(common[-1])
        assert list(a.t_sums) == al[r]["sums"], ("aligned", r)
        assert list(a.m_sums) == _exact_mem(kept[r], common), ("aligned mem sums (time kind)", r)
    if series:
        ser = torch.empty(16 * n, dtype=torch.float64, device="cuda")
        engines[0].win_reduce([e.win_rows_tensor(_abi.KIND_TIME, n) for e in engines],
                              _abi.MASK_TIME | _abi.MASK_MEM, n, 0, n, ser)
        torch.cuda.synchronize()
        ref = fast_oracle.series16(np.stack([a["rows"] for a in al]))
        np.testing.assert_array_equal(ser.view(16, n).cpu().numpy(), ref)
    return got


# ------------------------------------------------------------------------------------ window mode
# (family, R, W, history rows, ring slots or None = whole history)
WINDOW_CASES = [
    ("lognormal", 2, 1025, 1280, None),        # 1025 summation positions, pad 0: planned walk
    ("startup", 3, 1023, 1279, None),          # 1023 rows + pad 1 = 1024 positions: not planned
    ("giant", 2, 8192, 8192 + 77, None),       # pad 179
    ("startup", 2, 8192, 8192, None),          # pad 0
    ("sparse", 3, 8193, 12_000, 9_000),        # the ring (9 000 of 12 000 rows) wraps
    ("ties", 3, 131_072, 131_072 + 300, None),
    ("giant", 3, 131_072, 200_000, 150_001),   # ring wraps, window inside it
    ("sparse", 2, 131_072, 131_072, None),
    ("ties", 2, 1 << 20, (1 << 20) + 5, None),
    ("lognormal", 3, 1 << 20, (1 << 20) + 1000, (1 << 20) + 500),
]


@pytest.mark.parametrize("family,R,W,hist,ring", WINDOW_CASES)
def test_window_sums(cuda, family, R, W, hist, ring):
    from oracle import fast_oracle

    recs = [make_records(family, hist, target_of(r, W + R), seed=11 + r) for r in range(R)]
    kept = [rc[-(ring or hist):] for rc in recs]
    engines = _engines(recs, ring=ring)
    try:
        infos = [e.win_prepare(W) for e in engines]
        slow = [_slow_rows(e) for e in engines]
        for r in range(R):
            assert list(infos[r].t_sums) == fast_oracle.rank_part(kept[r], W)["sums"], ("window", family, r)
        print(f"[k3e slow rows] {family} R={R} W={W}: {slow}")
        if family == "startup":
            assert all(s > 0 for rank in slow for s in rank), slow
        if family == "giant":
            for r in range(R):
                chain = {0: 0, 2: 1, 3: 2, 4: 3, 5: 4}[target_of(r, W + R)]
                assert slow[r][chain] > 0, (r, slow)
        _check_aligned_time(engines, infos, kept, W)
    finally:
        _close(engines)


def test_stall_overflows_the_slot_table(cuda):
    """At least two chains per rank sit inside the plan's margin band for the whole 2^20-row
    window: more than XS_SLOT_CAP unsafe (chunk, chain) pairs, so the chunks left without a slot
    are walked from the rows (xs_walk_rows), and the walk's staging lists (XS_IG groups, XS_TS
    crossing chunks per batch) overflow to their on-demand fetches."""
    from oracle import fast_oracle

    W, hist = 1 << 20, (1 << 20) + 100
    targets = (0, 4)                   # dl (+ dl+traced), opt (+ traced, dl+traced)
    recs = [make_records("stall", hist, t, seed=5) for t in targets]
    pad = (256 - hist % 256) % 256
    for r in range(2):
        pairs = _band_pairs(_window_chains(recs[r], W), pad)
        assert pairs > XS_SLOT_CAP, (r, pairs)
    engines = _engines(recs)
    try:
        infos = [e.win_prepare(W) for e in engines]
        slow = [_slow_rows(e) for e in engines]
        print(f"[k3e slow rows] stall R=2 W={W}: {slow}")
        for r in range(2):
            assert list(infos[r].t_sums) == fast_oracle.rank_part(recs[r], W)["sums"], ("window", r)
        _check_aligned_time(engines, infos, recs, W)
    finally:
        _close(engines)


# ------------------------------------------------------------------------------------ aligned mode
@pytest.mark.parametrize("layout,family", [
    ("offset", "ties"),      # dense windows, step ids offset per rank: row source dense_first
    ("offset", "stall"),
    ("holes", "giant"),      # rank 1 has holes: rank 0's selection is scattered (gathered xrows),
    ("holes", "ties"),       # rank 1's own selection is contiguous (sel_rows[0])
])
def test_aligned_row_sources(cuda, layout, family):
    from oracle import fast_oracle
    from traceml_b200 import _abi

    R, S, W = 2, 150_000, 140_000
    recs = []
    for r in range(R):
        rc = make_records(family, S, target_of(r, 3), seed=21 + r, first_step=1 + (7 * r if layout == "offset" else 0))
        if layout == "holes" and r == 1:
            rng = np.random.default_rng(9)
            rc = np.delete(rc, np.sort(rng.choice(np.arange(10, S - 10), 3000, replace=False)))
        recs.append(rc)
    engines = _engines(recs)
    try:
        infos = [e.win_prepare(W) for e in engines]
        for r in range(R):
            assert list(infos[r].t_sums) == fast_oracle.rank_part(recs[r], W)["sums"], ("window", r)
        if layout == "offset":
            assert all(i.dense[_abi.KIND_TIME] for i in infos)
        else:
            assert infos[0].dense[_abi.KIND_TIME] and not infos[1].dense[_abi.KIND_TIME]
        got = _check_aligned_time(engines, infos, recs, W)
        # none of these windows is a rank's whole window: no rank may take the lock-step copy
        for r in range(R):
            assert int(got[r].n_common) < int(infos[r].n_cand[_abi.KIND_TIME]) or \
                int(got[r].start_step) != int(infos[r].lo[_abi.KIND_TIME])
    finally:
        _close(engines)


# ------------------------------------------------------------------------------------ world of one
@pytest.mark.parametrize("n", [1 << 17, (1 << 17) + 1])
def test_world_of_one(cuda, n):
    """One rank has nobody to break a tie against: up to 2^17 rows it still gets reference-order
    sums (bit for bit), above that the deterministic tree sums (rel 1e-9)."""
    from oracle import fast_oracle

    rec = make_records("ties", n, 2, seed=3)
    engines = _engines([rec])
    try:
        got = list(engines[0].win_prepare(n).t_sums)
        ref = fast_oracle.rank_part(rec, n)["sums"]
        if n <= 1 << 17:
            assert got == ref
        else:
            np.testing.assert_allclose(got, ref, rtol=1e-9, atol=0)
    finally:
        _close(engines)


# ------------------------------------------------------------------------------------ deferred job
@pytest.mark.parametrize("family", ["lognormal", "stall"])
def test_deferred_exact_sums(cuda, family):
    """``tml_win_set_defer``: win_prepare launches K3e on the side stream and returns tree sums; an
    aligned K3e on the main stream must wait for the shared workspace; tml_win_exact_collect then
    yields the window sums.  Both results bit for bit."""
    from oracle import fast_oracle
    from traceml_b200 import _abi

    lib = _abi.lib()
    R, S, W = 2, 300_000, 300_000
    recs = [make_records(family, S, target_of(r, 1), seed=31 + r, first_step=1 + 7 * r) for r in range(R)]
    engines = _engines(recs)
    try:
        for e in engines:
            _abi.check(lib.tml_win_set_defer(e.handle, 1), "tml_win_set_defer")
        infos = [e.win_prepare(W) for e in engines]
        for r in range(R):
            np.testing.assert_allclose(list(infos[r].t_sums), fast_oracle.rank_part(recs[r], W)["sums"],
                                       rtol=1e-9, atol=0)
        _check_aligned_time(engines, infos, recs, W, series=False)
        for r, e in enumerate(engines):
            out = (C.c_double * 7)()
            _abi.check(lib.tml_win_exact_collect(e.handle, None, out), "tml_win_exact_collect")
            assert list(out) == fast_oracle.rank_part(recs[r], W)["sums"], ("deferred window", r)
    finally:
        for e in engines:
            lib.tml_win_set_defer(e.handle, 0)
        _close(engines)


# ------------------------------------------------------------------------------------ > 1024 groups
def test_more_than_one_walk_batch(cuda):
    """2^23 + 2^20 rows: 1153 groups of 32 chunks, past the walk's 1024-group staging batch."""
    from oracle import fast_oracle

    W = (1 << 23) + (1 << 20)
    rec = make_records("ties", W + 100, 3, seed=41)
    engines = _engines([rec, rec])     # rank 1 replays rank 0's records (host memory)
    try:
        infos = [e.win_prepare(W) for e in engines]
        ref = fast_oracle.rank_part(rec, W)["sums"]
        print(f"[k3e slow rows] ties R=2 W={W}: {[_slow_rows(e) for e in engines]}")
        for r in range(2):
            assert list(infos[r].t_sums) == ref, ("window", r)
    finally:
        _close(engines)


# ------------------------------------------------------------------------------------ memory
def _halfway(rec, which, up):
    """Move the last row of ``which`` so that the column's exact sum lies halfway between two
    doubles: rounding to even goes down (``up`` False) or up."""
    tot = int(rec[which].sum(dtype=np.uint64))
    e = tot.bit_length() - 53                       # ulp of the sum = 2^e
    base = (tot >> e) << e
    if ((base >> e) & 1) != (1 if up else 0):       # an odd lower neighbour rounds up
        base += 1 << e
    target = base + (1 << (e - 1))
    rec[which][-1] = np.uint64(int(rec[which][-1]) + (target - tot))
    assert int(rec[which].sum(dtype=np.uint64)) == target and float(target) != target
    assert (float(target) > target) == up


@pytest.mark.parametrize("mem_holes", [False, True])
def test_memory_sums_above_2_53(cuda, mem_holes):
    """Peaks of 80-180 GB over 10^5 rows: the exact byte sums exceed 2^53 and are rounded once.
    Rank 0's sums lie exactly halfway between two doubles (alloc rounds down, resv up)."""
    from oracle import fast_oracle
    from traceml_b200 import _abi, sections

    import replay

    R, n, W = 2, 100_000, 100_000
    recs = [make_records("mem", n, target_of(r, 0), seed=51 + r) for r in range(R)]
    _halfway(recs[0], "peak_alloc", up=False)
    _halfway(recs[0], "peak_resv", up=True)
    if mem_holes:                      # rank 1 reports no memory on some steps: the kinds differ
        off = np.arange(100, n, 997)
        recs[1]["flags"][off] = 0
        recs[1]["peak_alloc"][off] = 0
        recs[1]["peak_resv"][off] = 0
    engines = _engines(recs)
    try:
        infos = [e.win_prepare(W) for e in engines]
        _check_aligned_time(engines, infos, recs, W)
        mem = [fast_oracle.mem_part(rc, W) for rc in recs]
        common = fast_oracle.common_suffix([m["steps"] for m in mem], W)
        got = _align(engines, infos, _abi.KIND_MEM, W)
        for r, a in enumerate(got):
            assert int(a.n_common) == common.size
            assert list(a.m_sums) == _exact_mem(recs[r], common), ("mem kind", r)
        res = sections.SummaryEngine(engines, ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=R).build(W, W)
        ref = fast_oracle.step_memory_section({r: recs[r] for r in range(R)}, window_size=W)
        assert plain(res["step_memory"]["per_global_rank"]) == plain(ref["per_global_rank"])
    finally:
        _close(engines)
