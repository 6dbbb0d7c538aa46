"""GPU: back-to-back native builds emit each build's sections text while the next build's pass runs.

``SummaryEngine.build`` returns sections whose JSON text is emitted from the result's own copy: by
the next build of the same ``SummaryEngine`` (while its window pass runs, or after its reduce on the
staged path), or on first access.  Whichever emits it, the text must be byte-identical to what a
build whose text is emitted on access gives, for chained and staged builds in any order.
"""
import pytest

S, W_BULK, W_SMALL, PROCS = 300_000, 300_000, 100_000, 60_000


@pytest.fixture(scope="module")
def engine():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    import replay
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=S + 8, proc_slots=65_536)
    eng.load_procs(replay.make_proc_replay("normal", 1, PROCS, seed=5)[0])
    eng.load_steps(replay.make_step_replay("input_straggler", 1, S, seed=7)[0])
    torch.cuda.synchronize()
    yield eng
    eng.close()


def _summary(eng):
    import replay
    from traceml_b200 import sections

    return sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1)


@pytest.mark.gpu
def test_deferred_text_equals_text_emitted_on_access(engine):
    windows = [W_BULK, W_BULK, W_SMALL, W_BULK, W_SMALL, W_SMALL, W_BULK]
    want = {}
    for w in set(windows):  # one build per SummaryEngine: its text is emitted on access
        res = _summary(engine).build(w, PROCS)
        want[w] = bytes(res.raw)
        assert bool(res["reduce"].fused_rows) == (w == W_BULK)
    summ = _summary(engine)
    got = [summ.build(w, PROCS) for w in windows]
    # every build but the last had its text emitted by the build after it
    assert all(r._raw is not None for r in got[:-1])
    assert got[-1]._raw is None
    for w, r in zip(windows, got):
        assert bytes(r.raw) == want[w]


@pytest.mark.gpu
def test_text_read_before_the_next_build_keeps_its_bytes(engine):
    summ = _summary(engine)
    first = summ.build(W_BULK, PROCS)
    text = bytes(first.raw)
    second = summ.build(W_BULK, PROCS)
    assert bytes(first.raw) == text == bytes(second.raw)
    assert first["step_time"]["data"]["aligned_window"]["steps_analyzed"] == W_BULK
