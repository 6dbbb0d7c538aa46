"""GPU: the chained single-rank build gives what the three-wait sequence gives.

With one rank and a bulk window, ``tml_reduce_run`` submits the fused window pass (which finalises
itself), the band sums and the process aggregates as one device submission with one copy and one
wait.  ``TML_FUSED_CHAIN=0`` keeps the older sequence (pass + k_finalize, wait; process aggregates,
wait; bands, wait).  The switch is read once per process, so each arm runs in a child process of its
own and the two are compared byte for byte: the sections' JSON text and the per-step series.

In one process (chained arm): builds that alternate with the staged path, which shares nothing
with the chained pass's accumulator, and a ring reset + reload must repeat their results exactly.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (scenario, steps, window, ring slots or None, process samples or None, fused expected)
CASES = {
    "dense": ("balanced", 300_000, 300_000, None, None, True),
    "straggler": ("input_straggler", 450_000, 300_000, None, None, True),
    "wrapped": ("balanced", 400_000, 400_000, 250_000, None, True),
    "duplicates": ("duplicates", 200_000, 200_000, None, None, False),   # not dense: staged fallback
    "below": ("balanced", 100_000, 100_000, None, None, False),          # below the bulk threshold
    "with_procs": ("balanced", 300_000, 300_000, None, 60_000, True),    # the process join on the device
    "nonmonotone": ("balanced", 200_000, 200_000, None, None, None),     # step ids decrease: an error
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

    scenario, S, W, ring, procs, _ = CASES[name]
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


def _child(name, out_dir):
    """Runs in a child process: one case under whatever TML_FUSED_CHAIN says, written to out_dir."""
    import torch

    torch.cuda.set_device(0)
    _, S, W, _, procs, _ = CASES[name]
    eng = _engine(name)
    meta = {"error": None}
    try:
        l0 = eng.launch_count
        raw, ser, mser, fused = _build(eng, W, procs or W)
        meta.update(launches=eng.launch_count - l0, fused=fused)
        with open(os.path.join(out_dir, "raw.json"), "wb") as fh:
            fh.write(raw)
        np.save(os.path.join(out_dir, "time.npy"), ser)
        np.save(os.path.join(out_dir, "mem.npy"), mser)
    except Exception as exc:  # noqa: BLE001 -- the error itself is the result
        meta["error"] = f"{type(exc).__name__}: {exc}"
    finally:
        eng.close()
    with open(os.path.join(out_dir, "meta.json"), "w") as fh:
        json.dump(meta, fh)


def _run_arm(name, chain, tmp_path):
    out = tmp_path / f"{name}_{chain}"
    out.mkdir()
    env = dict(os.environ, TML_FUSED_CHAIN=chain)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), name, str(out)]
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    with open(out / "meta.json") as fh:
        meta = json.load(fh)
    if meta["error"] is not None:
        return meta, None, None, None
    raw = (out / "raw.json").read_bytes()
    return meta, raw, np.load(out / "time.npy"), np.load(out / "mem.npy")


@pytest.fixture(scope="module")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chain_matches_three_wait_sequence(cuda, tmp_path, name):
    fused = CASES[name][5]
    m1, raw1, t1, g1 = _run_arm(name, "1", tmp_path)
    m0, raw0, t0, g0 = _run_arm(name, "0", tmp_path)
    if fused is None:  # a ring whose step ids decrease: the same error from both sequences
        assert m1["error"] is not None and "step ids decrease" in m1["error"], m1
        assert m1["error"] == m0["error"]
        return
    assert m1["error"] is None and m0["error"] is None, (m1, m0)
    assert m1["fused"] == m0["fused"] == fused
    assert raw1 == raw0
    assert t1.tobytes() == t0.tobytes() and t1.shape == t0.shape
    assert g1.tobytes() == g0.tobytes() and g1.shape == g0.shape
    if fused:  # the k_finalize launch behind the pass is gone, nothing else
        assert m0["launches"] - m1["launches"] == 1, (m0, m1)
    else:
        assert m0["launches"] == m1["launches"], (m0, m1)


@pytest.mark.gpu
def test_chain_interleaved_with_staged_and_reset(cuda):
    import replay
    from traceml_b200 import sections

    if os.environ.get("TML_FUSED_CHAIN", "1").startswith("0"):
        pytest.skip("the chained sequence is switched off in this process")
    _, S, W, _, procs, _ = CASES["with_procs"]
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


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _child(sys.argv[1], sys.argv[2])
