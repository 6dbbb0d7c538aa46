"""K3e arithmetic (csrc/tml_exact_sum.h) on the CPU: the reference's sequential ``s += x`` sums
reproduced BIT FOR BIT from composed integer maps -- plan, chunk / group composition, verified
application, 32-row tile fallback -- fuzzed against a plain sequential loop through the host
emulation ``tml_xs_host_sum`` (the kernels share the header; GPU runs: test_gpu_exact_sums.py,
test_gpu_parity_holes.py)."""
import ctypes as C

import numpy as np
import pytest

from traceml_b200 import _abi


def xs(x, planned=1):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out, slow = C.c_double(), C.c_uint64()
    rc = _abi.lib().tml_xs_host_sum(x.ctypes.data, len(x), planned, C.byref(out), C.byref(slow))
    assert rc == 0
    return out.value, slow.value


def seq(x):
    x = np.asarray(x, dtype=np.float64)
    return float(np.add.accumulate(x)[-1]) if len(x) else 0.0


def make(kind, n, rng):
    if kind == 0:
        return rng.integers(1, 40_000_000, n).astype(np.float64) / 1e6         # ns / 1e6: the real shape
    if kind == 1:
        return rng.uniform(0, 1, n) * 10.0 ** rng.integers(-12, 12, n)        # 24 decades of range
    if kind == 2:
        return rng.integers(0, 5, n).astype(np.float64) * 2.0 ** int(rng.integers(-3, 3))  # ties everywhere
    if kind == 3:
        return np.where(rng.uniform(size=n) < 0.5, 0.0, rng.uniform(0, 50, n))  # half the rows unused (+0.0)
    if kind == 4:
        return np.full(n, 0.5 ** int(rng.integers(0, 60)))                      # constant power of two
    if kind == 5:
        return rng.integers(0, 2 ** 20, n).astype(np.float64) * 2.0 ** -30 + 1.0
    if kind == 6:
        return np.concatenate([[1e18], rng.uniform(0, 1e3, n)])                 # one giant, then dust
    if kind == 8:  # stalled just below 2^e: every chunk lies inside the plan's 1e-6 margin band
        e = int(rng.integers(-10, 60))
        return np.concatenate([[2.0 ** e * (1.0 - 3.0e-7)], rng.uniform(1, 2, n) * 2.0 ** (e - 45)])
    if kind == 9:  # multiples of 1/64 near 2^40: past 2^47 every odd addend is an exact tie
        return rng.integers(2 ** 45, 2 ** 47, n).astype(np.float64) * 2.0 ** -6
    if kind == 10:  # giants inside 32-row tiles: the sum jumps several binades mid-tile
        x = rng.uniform(1, 3, n)
        for j, t in enumerate(sorted(rng.choice(max(1, n // 32), 3, replace=True))):
            x[min(n - 1, 32 * int(t) + 13)] = 10.0 ** (3 * j + 4)
        return x
    return rng.lognormal(2, 3, n)


@pytest.mark.parametrize("kind", range(11))
def test_bit_exact_against_sequential_loop(kind):
    rng = np.random.default_rng(100 + kind)
    for _ in range(40):
        n = int(rng.integers(1, 30_000))
        x = make(kind, n, rng)
        ref = seq(x)
        for planned in (0, 1):
            got, _ = xs(x, planned)
            assert got == ref, (kind, n, planned, got, ref)


def test_bench_sized_chain_needs_almost_no_sequential_adds():
    rng = np.random.default_rng(7)
    x = rng.integers(30_000_000, 45_000_000, 4_000_000).astype(np.float64) / 1e6
    got, slow = xs(x, 1)
    assert got == seq(x)
    assert slow <= 64 * 32, slow   # one 32-row tile per binade crossing (~26 of them) + start-up


def test_python_loop_is_the_same_thing():
    """np.add.accumulate == the reference's Python ``s += x`` loop (the oracle's own pin)."""
    rng = np.random.default_rng(3)
    x = rng.uniform(0, 40, 50_000)
    s = 0.0
    for v in x.tolist():
        s += v
    assert seq(x) == s == xs(x)[0]


def test_empty_and_zero_chains():
    assert xs(np.zeros(0))[0] == 0.0
    assert xs(np.zeros(5000)) == (0.0, 0)


# ---------------------------------------------------------------------------------------------
# Executable specification of the walk's warp-wide map application (tml_exact_sum.cuh:
# xs_apply_run).  The kernel applies 32 maps per step: lane i composes entries j..j+i by an
# inclusive scan, applies that prefix to the running significand and the warp keeps the longest
# prefix that stays inside the binade.  The GPU tests check the kernel's sums; this checks the
# algorithm -- on Python integers, lane by lane -- against applying the entries one after the other.
_ZERO = -2          # XS_PLAN_ZERO
_INVALID = 2 ** 64 - 1


def _apply_sequential(S, eb, f, e, j, end):
    while j < end:
        E = e[j]
        if E == _ZERO:
            j += 1
            continue
        if E != eb or E < 1:
            break
        c0, c1 = f[j]
        S2 = S + (c1 if S & 1 else c0)
        if c0 == _INVALID or (S2 >> 53):
            break
        S, j = S2, j + 1
    return S, j


def _compose(f, g):  # f first, then g (xs_compose_raw)
    return (f[0] + (g[1] if f[0] & 1 else g[0]), f[1] + (g[1] if (1 + f[1]) & 1 else g[0]))


def _apply_warp(S, eb, f, e, j, end):
    while j < end:
        maps, ok = [], []
        for lane in range(32):
            idx = j + lane
            E, m = (e[idx], f[idx]) if idx < end else (_ZERO, (0, 0))
            zero = E == _ZERO
            ok.append(zero or (E == eb and 1 <= E < 0x7ff and m[0] != _INVALID))
            maps.append((0, 0) if zero else m)
        nvalid = next((i for i, o in enumerate(ok) if not o), 32)
        maps = [m if i < nvalid else (0, 0) for i, m in enumerate(maps)]
        d = 1
        while d < 32:  # Hillis-Steele inclusive scan, ordered composition
            maps = [_compose(maps[i - d], maps[i]) if i >= d else maps[i] for i in range(32)]
            d *= 2
        Si = [S + (p[1] if S & 1 else p[0]) for p in maps]
        napply = min(next((i for i, s in enumerate(Si) if s >> 53), 32), nvalid)
        if napply:
            S = Si[napply - 1]
        j += napply
        if napply < 32:
            break
    return S, min(j, end)


def test_warp_wide_application_equals_one_by_one():
    import random

    rnd = random.Random(7)
    for _ in range(4000):
        n, eb = rnd.randint(1, 100), rnd.choice([0, 5, 1000])
        f, e = [], []
        for _ in range(n):
            r = rnd.random()
            if r < 0.10:
                e.append(_ZERO); f.append((7, 7))
            elif r < 0.13:
                e.append(rnd.choice([-1, -3, -10, eb + 1 if eb else 3])); f.append((1, 1))
            elif r < 0.15:
                e.append(eb); f.append((_INVALID, _INVALID))
            else:
                q = rnd.randint(0, 2 ** 50 if rnd.random() < 0.05 else 2 ** 40)
                e.append(eb); f.append(rnd.choice([(q, q), (q + (q & 1), q + ((q + 1) & 1))]))
        S, j0 = rnd.randint(2 ** 52, 2 ** 53 - 1), rnd.randint(0, n - 1)
        assert _apply_sequential(S, eb, f, e, j0, n) == _apply_warp(S, eb, f, e, j0, n)


def test_transposed_butterfly_totals_land_on_every_fourth_lane():
    """K3a's chunk-sum reduction (tml_engine.cu, ``if (csum)``): 8 values per lane are folded
    8 -> 4 -> 2 -> 1 while lanes pair up over bits 4, 3, 2, then two plain levels over bits 1, 0;
    lane 4 j must end up with the total of value j over the 32 lanes (9 exchanges instead of 35)."""
    rng = np.random.default_rng(0)
    V = rng.integers(0, 1000, size=(32, 8)).astype(np.float64)
    V[:, 7] = 0.0
    lanes = np.arange(32)
    v = V.copy()
    for bit, width in ((16, 4), (8, 2), (4, 1)):
        hi = (lanes & bit) != 0
        nv = v.copy()
        for i in range(width):
            keep = np.where(hi, v[:, i + width], v[:, i])
            send = np.where(hi, v[:, i], v[:, i + width])
            nv[:, i] = keep + send[lanes ^ bit]
        v = nv
    t = v[:, 0]
    t = t + t[lanes ^ 2]
    t = t + t[lanes ^ 1]
    for j in range(8):
        assert t[4 * j] == V[:, j].sum()
