"""GPU: the single-rank bulk build's paired series.

With one rank the median and the worst series of a metric hold the same values, so the bulk build
stores each pair once -- 8 physical rows, row m mapped at rows 2m and 2m+1 of a 16-row address range
-- and the window pass writes 64 B per step instead of 128.  Consumers see a [16, n] view with row
stride ``ld`` (n rounded up to the 2 MiB mapping granularity).  Checked here:

* at window sizes on either side of the granularity (n * 8 below, at and above 2 MiB) up to 4·10⁶:
  the series, bit for bit, against ``oracle.fast_oracle.series16`` and against what the public
  ``tml_win_fused`` writes into a plain 16-row buffer; the band sums and tails against
  ``tml_win_bands`` over that plain buffer; and up to 2^18 steps the sections against the row-level
  oracles;
* the view: its stride, its aliasing (a write into row 0 shows in row 1), one buffer for both
  sections;
* sequences in one context: dense, staged (a window that is not dense), dense again; a larger window
  that remaps the range, then a smaller one; a wrapped ring; reset and reload; clones of the view;
* no device memory left behind after 30 contexts that each remap and close;
* ``TML_SERIES_ALIAS=0`` in a process of its own: the plain buffer, with the same series bytes,
  sections JSON and kernel launches per build.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import build_vs_row_oracles

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAN = 2 << 20  # device-memory mapping granularity of an H100, bytes
SIZES = [(1 << 17) + 1, 262_144, 262_145, 3 * 262_144 - 1, 1_000_000, 4_000_000]
ROW_ORACLE_MAX = 1 << 18  # the row-level oracles take minutes above it; the band sums are checked instead


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _recs(scenario, n, seed):
    import replay

    return replay.make_step_replay(scenario, 1, n, seed=seed)[0]


def _engine(recs, slots=None):
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=slots or len(recs) + 8, proc_slots=64)
    eng.load_steps(recs)
    torch.cuda.synchronize()
    return eng


def _build(eng, W):
    import replay
    from traceml_b200 import sections

    return sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, W)


def _expected(retained, W):
    """The series of a dense window: its aligned rows are the ring's last W records."""
    from oracle import fast_oracle as fo

    return fo.series16(fo.window_rows(retained[-W:])[None])


def _time_rows(retained, W):
    """The aligned time rows of any window: the oldest usable row of each step id among the last W."""
    from oracle import fast_oracle as fo

    win = retained[-W:]
    rows = fo.window_rows(win)
    usable = np.nonzero((rows[:, [fo.C_DL, fo.C_FWD, fo.C_BWD, fo.C_OPT, fo.C_WALL]] > 0).any(axis=1))[0]
    _, first = np.unique(win["step"][usable], return_index=True)
    return rows[usable[first]]


def _public_fused(eng, W, n):
    """What the public tml_win_fused writes into a plain [16, n] buffer (device)."""
    from traceml_b200 import _abi

    buf = torch.empty(16 * n, dtype=torch.float64, device="cuda")
    info, al, ok = _abi.WinInfo(), _abi.AlignInfo(), C.c_uint32(7)
    rc = _abi.lib().tml_win_fused(eng.handle, int(W), buf.data_ptr(), 0, C.byref(info), C.byref(al), C.byref(ok))
    torch.cuda.synchronize()
    assert rc == 0 and ok.value == 1, _abi.lib().tml_last_error()
    return buf.view(16, n)


def _plain_bands(eng, plain, n):
    """tml_win_bands over a plain 16-row series, with the layout the single-rank build uses."""
    from traceml_b200 import _abi
    from traceml_b200.reduce import trend_layout

    a = _abi.BandArgs()
    a.n_common, a.shard_lo, a.shard_hi = n, 0, n
    layouts = (trend_layout(n, min_points=200, warmup_frac=0.10), trend_layout(n, min_points=50, warmup_frac=0.0))
    for k, lay in enumerate(layouts):
        for b in range(3):
            a.band_lo[k][b], a.band_hi[k][b] = (lay[b] if lay else (0, 0))
    a.tail_first[0], a.tail_first[1] = 0, n - min(n, 1000)
    out = eng.win_bands(plain, a)
    return ([[out.sum[s][b] for b in range(3)] for s in range(16)], [[out.cnt[s][b] for b in range(3)] for s in range(16)],
            list(out.tail_first), list(out.tail_last))


def _check_paired(red, n):
    """The build took the paired path: a [16, n] view with row stride ld, one buffer for both sections."""
    s = red.time.series
    ld = s.stride(0)
    assert red.fused_rows and red.series_paired
    assert tuple(s.shape) == (16, n) and s.stride() == (ld, 1)
    assert ld >= n and (ld * 8) % GRAN == 0
    assert red.mem.series.data_ptr() == s.data_ptr()
    return ld


# ----------------------------------------------------------------------------- 1. results
@pytest.mark.parametrize("n", SIZES)
def test_paired_series_vs_oracles(cuda, n):
    recs = _recs("balanced", n, seed=11)
    eng = _engine(recs)
    try:
        got = build_vs_row_oracles(eng, recs, n) if n <= ROW_ORACLE_MAX else _build(eng, n)
        red = got["reduce"]
        assert _check_paired(red, n) * 8 == -(-n * 8 // GRAN) * GRAN   # a fresh context: n rounded up
        exp = _expected(recs, n)
        t = red.time.series.cpu().numpy()
        m = red.mem.series.cpu().numpy()
        assert t.tobytes() == exp.tobytes() and m.tobytes() == exp.tobytes()
        k = red.time
        plain = _public_fused(eng, n, n)
        assert plain.cpu().numpy().tobytes() == t.tobytes()
        # k_bands read the paired rows at stride ld: the same bits as over the plain rows
        got = (k.band_sum, k.band_cnt, list(k.tail_first), list(k.tail_last))
        for a, b in zip(got, _plain_bands(eng, plain, n)):
            assert np.array(a, dtype=np.float64).tobytes() == np.array(b, dtype=np.float64).tobytes()
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 2. the view
def test_paired_view_aliases_its_rows(cuda):
    n = 262_145
    recs = _recs("balanced", n, seed=12)
    eng = _engine(recs)
    try:
        red = _build(eng, n)["reduce"]
        _check_paired(red, n)
        s = red.time.series
        before = s[:, :2].cpu().numpy()
        assert (before[0::2] == before[1::2]).all()
        s[0, 0] = -12345.5
        torch.cuda.synchronize()
        after = s[:, :2].cpu().numpy()
        assert after[0, 0] == -12345.5 and after[1, 0] == -12345.5   # one physical row, two addresses
        assert after[2:].tobytes() == before[2:].tobytes() and after[:2, 1].tobytes() == before[:2, 1].tobytes()
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 3. sequences
def test_dense_staged_dense(cuda):
    """A window that is not dense takes the staged path into its own 16-row buffer; the paired range
    the dense builds around it use is untouched by it."""
    from oracle import fast_oracle as fo

    n = 300_000
    dense = _recs("balanced", n, seed=13)
    dups = _recs("duplicates", 200_000, seed=14)
    eng = _engine(dense, slots=n + 8)
    try:
        exp = _expected(dense, n)
        first = _build(eng, n)["reduce"]
        _check_paired(first, n)
        assert first.time.series.cpu().numpy().tobytes() == exp.tobytes()

        eng.reset()
        eng.load_steps(dups)
        torch.cuda.synchronize()
        staged = _build(eng, 200_000)["reduce"]
        assert not staged.fused_rows and not staged.series_paired
        s = staged.time.series
        rows = _time_rows(dups, 200_000)
        assert tuple(s.shape) == (16, len(rows)) and s.stride() == (len(rows), 1)
        assert s[:12].cpu().numpy().tobytes() == fo.series16(rows[None])[:12].tobytes()

        eng.reset()
        eng.load_steps(dense)
        torch.cuda.synchronize()
        again = _build(eng, n)["reduce"]
        _check_paired(again, n)
        assert again.time.series.cpu().numpy().tobytes() == exp.tobytes()
    finally:
        eng.close()


def test_remap_wrap_reset_and_clone(cuda):
    S, slots = 1_300_000, 1_100_000      # the ring wraps: the window's first row is not slot 0
    recs = _recs("balanced", S, seed=15)
    retained = recs[-slots:]
    eng = _engine(recs, slots=slots)
    try:
        small = _build(eng, 300_000)["reduce"]
        ld_small = _check_paired(small, 300_000)
        keep = small.time.series.clone()
        assert keep.cpu().numpy().tobytes() == _expected(retained, 300_000).tobytes()

        big = _build(eng, 1_000_000)["reduce"]          # needs a larger row stride: remapped
        ld_big = _check_paired(big, 1_000_000)
        assert ld_big > ld_small
        assert big.time.series.cpu().numpy().tobytes() == _expected(retained, 1_000_000).tobytes()

        for W in (300_000, 1_000_000 - 1):              # t_start > 0 in a wrapped ring; the range only grows
            red = _build(eng, W)["reduce"]
            assert _check_paired(red, W) == ld_big
            assert red.time.series.cpu().numpy().tobytes() == _expected(retained, W).tobytes()
        assert keep.cpu().numpy().tobytes() == _expected(retained, 300_000).tobytes()  # the clone is its own

        eng.reset()
        eng.load_steps(recs)
        torch.cuda.synchronize()
        red = _build(eng, 300_000)["reduce"]
        _check_paired(red, 300_000)
        assert red.time.series.cpu().numpy().tobytes() == keep.cpu().numpy().tobytes()
    finally:
        eng.close()


# ----------------------------------------------------------------------------- 4. no leak
def test_remap_and_close_leave_no_memory_behind(cuda):
    recs = _recs("balanced", 1_000_000, seed=16)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(30):
        eng = _engine(recs)
        try:
            for W in (300_000, 1_000_000, 300_000):    # the second build remaps the range
                assert _build(eng, W)["reduce"].series_paired
        finally:
            eng.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert free0 - torch.cuda.mem_get_info()[0] < 64 << 20


# ----------------------------------------------------------------------------- 5. the plain buffer
FALLBACK_N = (262_145, 300_000)


def _fingerprint(sizes=FALLBACK_N):
    """Per window size: what a build hands back, hashed (run in a process of its own)."""
    torch.cuda.set_device(0)
    out = []
    for n in sizes:
        eng = _engine(_recs("balanced", n, seed=17))
        try:
            _build(eng, n)
            l0 = eng.launch_count
            res = _build(eng, n)
            red = res["reduce"]
            out.append({"n": n, "paired": bool(red.series_paired), "ld": red.time.series.stride(0),
                        "launches": eng.launch_count - l0,
                        "series": hashlib.sha256(red.time.series.cpu().numpy().tobytes()).hexdigest(),
                        "sections": hashlib.sha256(bytes(res.raw)).hexdigest()})
        finally:
            eng.close()
    return out


CHILD = """
import json, os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import test_gpu_series_alias as t
print("FINGERPRINT", json.dumps(t._fingerprint()))
"""


def _child(alias):
    env = dict(os.environ, TML_SERIES_ALIAS=alias)
    p = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-3000:])
    line = [x for x in p.stdout.splitlines() if x.startswith("FINGERPRINT ")][-1]
    return json.loads(line[len("FINGERPRINT "):])


def test_plain_buffer_switch(cuda):
    plain, paired = _child("0"), _child("1")
    for a, b in zip(plain, paired):
        assert not a["paired"] and a["ld"] == a["n"]
        assert b["paired"] and b["ld"] * 8 % GRAN == 0
        assert a["series"] == b["series"] and a["sections"] == b["sections"]
        assert a["launches"] == b["launches"] == 2
