"""GPU: the single-rank build against the oracles.

With one rank and a bulk window, ``tml_reduce_run`` submits the fused window pass (which finalises
itself), the band sums and the process aggregates as one device submission with one copy and one
wait; a window that is not dense, or not above 2^17 rows, takes the staged path.  Every case builds
once with the native driver and checks the per-step series bit for bit against
``oracle.fast_oracle.series16`` over the aligned window, the step-time and step-memory sections
against the row-level oracles, and the kernels launched per build.

In one process: builds that alternate with the staged path, which shares nothing with the chained
pass's accumulator, and a ring reset + reload must repeat their results exactly.
"""
import numpy as np
import pytest

from helpers import build_vs_row_oracles

# name: (scenario, steps, window, ring slots or None, process samples or None, fused expected,
#        kernels launched per build)
CASES = {
    "dense": ("balanced", 300_000, 300_000, None, None, True, 2),
    "straggler": ("input_straggler", 450_000, 300_000, None, None, True, 2),
    "wrapped": ("balanced", 400_000, 400_000, 250_000, None, True, 2),
    "duplicates": ("duplicates", 200_000, 200_000, None, None, False, 22),   # not dense: staged fallback
    "below": ("balanced", 100_000, 100_000, None, None, False, 9),           # below the bulk threshold
    "with_procs": ("balanced", 300_000, 300_000, None, 60_000, True, 5),     # the process join on the device
    "nonmonotone": ("balanced", 200_000, 200_000, None, None, None, None),   # step ids decrease: an error
}
PROC_SLOTS = 65_536


def _records(scenario, S, nonmonotone=False):
    import replay

    recs = replay.make_step_replay(scenario, 1, S, seed=77)[0]
    if nonmonotone:
        recs = recs.copy()
        recs["step"][150_000], recs["step"][150_001] = recs["step"][150_001], recs["step"][150_000]
    return recs


def _engine(name):
    import replay
    import torch
    from traceml_b200.engine import Engine

    scenario, S, W, ring, procs, _, _ = CASES[name]
    eng = Engine(device=0, rank=0, world=1, ring_slots=ring or (S + 8), proc_slots=PROC_SLOTS)
    if procs:
        eng.load_procs(replay.make_proc_replay("normal", 1, procs, seed=5)[0])
    eng.load_steps(_records(scenario, S, nonmonotone=name == "nonmonotone"))
    torch.cuda.synchronize()
    return eng


def _build(eng, W, proc_rows):
    """One native build: (raw JSON bytes, time series, memory series, fused?)"""
    import replay
    from traceml_b200 import sections

    res = sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1).build(W, proc_rows)
    red = res["reduce"]
    return (bytes(res.raw), red.time.series.cpu().numpy().copy(), red.mem.series.cpu().numpy().copy(),
            bool(red.fused_rows))


def _aligned_rows(recs, W):
    """One rank's aligned windows as WindowRows in step order: time (the oldest usable row of each step
    id among the last W rows) and memory (the newest row with memory of each step id, newest W ids)."""
    from oracle import fast_oracle as fo

    win = recs[-W:]
    rows = fo.window_rows(win)
    usable = np.nonzero((rows[:, [fo.C_DL, fo.C_FWD, fo.C_BWD, fo.C_OPT, fo.C_WALL]] > 0).any(axis=1))[0]
    _, first = np.unique(win["step"][usable], return_index=True)
    mem = recs[(recs["flags"] & fo.FLAG_HAS_MEM) != 0]
    _, last = np.unique(mem["step"][::-1], return_index=True)
    return rows[usable[first]][-W:], fo.window_rows(mem[len(mem) - 1 - last])[-W:]


@pytest.fixture(scope="module")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_single_rank_build_vs_oracles(cuda, name):
    from oracle import fast_oracle
    from traceml_b200 import _abi

    scenario, S, W, ring, procs, fused, launches = CASES[name]
    eng = _engine(name)
    try:
        if fused is None:  # a ring whose step ids decrease (one place)
            with pytest.raises(_abi.TraceMLNativeError, match=r"step ids decrease.*\(1 places\)"):
                _build(eng, W, W)
            return
        retained = _records(scenario, S)[-(ring or S + 8):]
        l0 = eng.launch_count
        got = build_vs_row_oracles(eng, retained, W, procs or W)
        assert eng.launch_count - l0 == launches
        red = got["reduce"]
        assert red.fused_rows == fused
        t_rows, m_rows = _aligned_rows(retained, W)
        # one K4 pass serves both sections when their aligned windows cover the same steps: the
        # memory series then comes from the time window's rows
        exp_t = fast_oracle.series16(t_rows[None])
        exp_m = fast_oracle.series16((t_rows if red.fused_pass else m_rows)[None])
        t = red.time.series.cpu().numpy()
        m = red.mem.series.cpu().numpy()
        assert t.shape == exp_t.shape and t[:12].tobytes() == exp_t[:12].tobytes()
        assert m.shape == exp_m.shape and m[12:16].tobytes() == exp_m[12:16].tobytes()
    finally:
        eng.close()


@pytest.mark.gpu
def test_chain_interleaved_with_staged_and_reset(cuda):
    import replay
    from traceml_b200 import sections

    _, S, W, _, procs, _, _ = CASES["with_procs"]
    eng = _engine("with_procs")
    try:
        first = _build(eng, W, procs)
        assert first[3]
        small = _build(eng, 100_000, procs)      # staged: K3a's accumulator, reference-order sums
        assert not small[3]
        again = _build(eng, W, procs)
        staged = sections.SummaryEngine([eng], native=False, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                        gpu_count=1).build(W, procs)   # the Python-sequenced stages
        assert staged["reduce"].time.series is not None
        third = _build(eng, W, procs)
        small2 = _build(eng, 100_000, procs)
        for got in (again, third):
            assert got[0] == first[0]
            assert got[1].tobytes() == first[1].tobytes() and got[2].tobytes() == first[2].tobytes()
        assert small2[0] == small[0] and small2[1].tobytes() == small[1].tobytes()
        # the bench's end-to-end leg: reset the rings, reload them, build
        eng.reset()
        eng.load_procs(replay.make_proc_replay("normal", 1, procs, seed=5)[0])
        eng.load_steps(_records("balanced", S))
        reloaded = _build(eng, W, procs)
        assert reloaded[0] == first[0]
        assert reloaded[1].tobytes() == first[1].tobytes() and reloaded[2].tobytes() == first[2].tobytes()
    finally:
        eng.close()
