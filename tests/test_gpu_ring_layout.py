"""GPU: the step ring's device layout.

The device keeps each 128-B ``tml_step_record`` as a 64-B hot half (what the window pass reads), a
64-B cold half and a memory byte (a copy of ``TML_REC_HAS_MEM``).  Checked here:

* records committed through the step path and drained are the public records the calls describe,
  byte for byte: mixed memory flags, call counts, host stamps and sequence numbers, across ring wraps;
* ``tml_ring_load`` from pageable and from pinned memory splits the public records into the ring and
  they read back byte for byte, at the staging chunk's edges, over several chunks, with a ring wrap
  inside a chunk and with more records than slots;
* windows whose oldest rows (or rows at tile edges and at the ring seam) lack memory build the
  sections of the row-level oracles;
* the chained single-rank build over a ring loaded through chunks with a wrap inside one equals the
  Python-sequenced staged build and the oracles.
"""
import time

import numpy as np
import pytest
import torch

from helpers import build_vs_row_oracles

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _chunk():
    from traceml_b200 import _abi

    return int(_abi.lib().tml_ring_load_chunk_())


def _read_ring(eng, first, n):
    """Records [first, first + n) of eng's ring, rebuilt in the public layout."""
    from traceml_b200 import _abi
    from traceml_b200.records import STEP_RECORD_DTYPE

    out = torch.empty(n * 128, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    _abi.check(_abi.lib().tml_ring_read_(eng.handle, first, n, out.data_ptr(), s), "tml_ring_read_")
    torch.cuda.synchronize()
    return out.cpu().numpy().view(STEP_RECORD_DTYPE)


def _random_records(n, seed):
    """Arbitrary bytes in every field, the memory bit set on about half the records."""
    from traceml_b200.records import STEP_RECORD_DTYPE

    rng = np.random.default_rng(seed)
    recs = rng.integers(0, 256, size=n * 128, dtype=np.uint8).view(STEP_RECORD_DTYPE)
    return recs


def test_commit_drain_bytes(cuda):
    from traceml_b200.engine import Engine
    from traceml_b200.records import STEP_RECORD_DTYPE

    slots = 37
    eng = Engine(device=0, ring_slots=slots)
    s = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(3)
    want = np.zeros(150, dtype=STEP_RECORD_DTYPE)
    got = []
    try:
        for k in range(150):
            for p in range(6):
                for _ in range(int(rng.integers(0, 3))):
                    d = int(rng.integers(1, 1 << 40))
                    eng.phase_host(p, d)
                    want["dur_ns"][k, p] += d
                    want["n_calls"][k, p] += 1
            flags = int(rng.integers(0, 1 << 32)) | (k % 3 == 0)
            if k % 5 == 0:
                flags &= ~1
            want["step"][k] = 1000 + k // 2  # repeated step ids
            want["peak_alloc"][k], want["peak_resv"][k] = rng.integers(0, 1 << 62, size=2)
            want["flags"][k] = flags
            want["host_ts"][k] = time.time() + k * 1e-3
            want["seq"][k] = k
            w = want[k]
            assert eng.step_commit(int(w["step"]), int(w["peak_alloc"]), int(w["peak_resv"]), int(w["flags"]),
                                   float(w["host_ts"]), s) == 0
            if k % 10 == 9:
                torch.cuda.synchronize()
                recs, dropped = eng.drain()
                assert dropped == 0
                got.append(recs.copy())
        got = np.concatenate(got)
        assert len(got) == 150
        assert got.tobytes() == want.tobytes()
        # what the ring holds now is the same, rebuilt from its halves
        assert _read_ring(eng, 150 - slots, slots).tobytes() == want[-slots:].tobytes()
    finally:
        eng.close()


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("size", ["chunk-1", "chunk", "chunk+1", "3chunks+5"])
def test_ring_load_roundtrip(cuda, pinned, size):
    from traceml_b200.engine import Engine

    ch = _chunk()
    n = {"chunk-1": ch - 1, "chunk": ch, "chunk+1": ch + 1, "3chunks+5": 3 * ch + 5}[size]
    lead = _random_records(50, seed=1)
    recs = _random_records(n, seed=2)
    eng = Engine(device=0, ring_slots=n + 100, proc_slots=64)
    try:
        eng.load_steps(lead)  # the bulk load starts at slot 50
        s = torch.cuda.current_stream().cuda_stream
        if pinned:
            host = torch.from_numpy(recs.view(np.uint8)).pin_memory()
            eng.load_steps_ptr(host.data_ptr(), n, s)
        else:
            eng.load_steps(recs, s)
        torch.cuda.synchronize()
        assert eng.step_count == 50 + n
        back = _read_ring(eng, 0, 50 + n)
        assert back[:50].tobytes() == lead.tobytes()
        assert back[50:].tobytes() == recs.tobytes()
    finally:
        eng.close()


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_ring_load_wraps_inside_a_chunk(cuda, pinned):
    """More records than slots: the last `slots` survive, the ring seam inside the first chunk."""
    from traceml_b200.engine import Engine

    ch = _chunk()
    slots = ch + 1000
    lead = _random_records(700, seed=4)
    recs = _random_records(2 * ch + 10, seed=5)
    eng = Engine(device=0, ring_slots=slots, proc_slots=64)
    try:
        eng.load_steps(lead)
        if pinned:
            host = torch.from_numpy(recs.view(np.uint8)).pin_memory()
            eng.load_steps_ptr(host.data_ptr(), len(recs), torch.cuda.current_stream().cuda_stream)
        else:
            eng.load_steps(recs)
        torch.cuda.synchronize()
        total = 700 + len(recs)
        assert _read_ring(eng, total - slots, slots).tobytes() == recs[-slots:].tobytes()
        # one record more: the seam moves by one
        extra = _random_records(1, seed=6)
        eng.load_steps(extra)
        torch.cuda.synchronize()
        back = _read_ring(eng, total + 1 - slots, slots)
        assert back[:-1].tobytes() == recs[-slots + 1:].tobytes() and back[-1:].tobytes() == extra.tobytes()
    finally:
        eng.close()


def _mem_holes(recs, rows):
    recs = recs.copy()
    recs["flags"][rows] &= ~np.uint32(1)
    recs["peak_alloc"][rows] = 0
    recs["peak_resv"][rows] = 0
    return recs


@pytest.mark.parametrize("case", ["oldest", "tile_edges", "seam"])
def test_window_rows_without_memory(cuda, case):
    """Rows lacking memory where the pass reads its neighbours from the ring (tile edges, seam)."""
    import replay
    from traceml_b200.engine import Engine

    S, W = 300_000, 300_000
    recs = replay.make_step_replay("balanced", 1, S, seed=11)[0]
    slots = S + 8
    if case == "oldest":
        rows = np.arange(0, 5_000)
    elif case == "tile_edges":
        rows = np.concatenate([np.arange(31, S, 4096), np.arange(32, S, 4099), np.arange(63, S, 8191)])
    else:
        slots = 250_000  # the last 250 000 records survive, from slot 50 000: the seam at retained row 200 000
        rows = np.array([S - slots + k for k in (0, 1, 199_999, 200_000, 200_001, 200_002)])
    recs = _mem_holes(recs, rows)
    eng = Engine(device=0, rank=0, world=1, ring_slots=slots, proc_slots=64)
    try:
        eng.load_steps(recs)
        torch.cuda.synchronize()
        build_vs_row_oracles(eng, recs[-min(slots, S):], min(W, slots))
    finally:
        eng.close()


def test_chain_equals_staged_after_chunked_wrapped_load(cuda):
    import replay
    from traceml_b200 import sections
    from traceml_b200.engine import Engine

    ch = _chunk()
    slots = ch + 40_000
    S = 2 * ch + 7_000
    recs = replay.make_step_replay("input_straggler", 1, S, seed=21)[0]
    eng = Engine(device=0, rank=0, world=1, ring_slots=slots, proc_slots=64)
    try:
        eng.load_steps(recs)
        torch.cuda.synchronize()
        kept = recs[-slots:]
        chained = build_vs_row_oracles(eng, kept, slots)
        red = chained["reduce"]
        assert red.fused_rows
        series = (red.time.series.cpu().numpy().copy(), red.mem.series.cpu().numpy().copy())
        staged = sections.SummaryEngine([eng], native=False, ram_total=replay.PROC_RAM_TOTAL_BYTES,
                                        gpu_count=1).build(slots, slots)["reduce"]
        assert staged.time.series.cpu().numpy().tobytes() == series[0].tobytes()
        assert staged.mem.series.cpu().numpy().tobytes() == series[1].tobytes()
    finally:
        eng.close()

