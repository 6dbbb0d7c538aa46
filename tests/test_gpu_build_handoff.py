"""GPU: back-to-back single-rank builds hand their results over without a copy.

The chained build's ``k_bands`` writes the pass's results into the context's pinned page, and
``SummaryEngine.build`` has the native driver write into the ``ReduceRunOut`` its result owns.  For
builds of one ``SummaryEngine`` with ring loads, host commits and a ring reset between them, each
build must equal a fresh ``SummaryEngine``'s build of the same ring: sections text (the reused
engine's emitted by the build after it), band sums and tails, process aggregates, alignment and the
series bit for bit; for packed windows, certified windows that stream the hot halves, and a context
without process samples (no process kernels, nothing to order in front of the bands).  A result kept
across later builds keeps its struct, its text and its ``timings_ms``.
"""
import pytest
import torch

import test_gpu_dense_certificate as dc
import test_gpu_packed_ring as pr

pytestmark = pytest.mark.gpu

SLOTS, W, PROCS = 300_000, 200_000, 3_000


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _engine(procs: bool):
    import replay
    from traceml_b200.engine import Engine

    eng = Engine(device=0, rank=0, world=1, ring_slots=SLOTS, proc_slots=4096)
    if procs:
        eng.load_procs(replay.make_proc_replay("normal", 1, PROCS, seed=9)[0])
    return eng


def _summary(eng):
    import replay
    from traceml_b200 import sections

    return sections.SummaryEngine([eng], ram_total=replay.PROC_RAM_TOTAL_BYTES, gpu_count=1)


def _facts(res):
    """What a build computed, as host values; the series cloned before any later build reuses them."""
    red = res["reduce"]
    o = red.out
    k = o.time
    return {"fused_rows": bool(red.fused_rows), "n_common": int(k.n_common),
            "steps": (int(k.start_step), int(k.end_step)), "n_rows": int(k.n_rows[0]),
            "t_sums": bytes(k.t_sums), "m_sums": bytes(k.m_sums),
            "band_sum": bytes(k.band_sum), "band_cnt": bytes(k.band_cnt),
            "tails": bytes(k.tail_first) + bytes(k.tail_last),
            "mem_bands": bytes(o.mem.band_sum) + bytes(o.mem.tail_first) + bytes(o.mem.tail_last),
            "procs": bytes(o.procs[0]),
            "series": red.time.series.clone() if red.time.series is not None else None}


def _fresh(eng):
    res = _summary(eng).build(W, PROCS)
    return _facts(res), bytes(res.raw)


def _same(got, want):
    for key in want:
        if key == "series":
            assert (got[key] is None) == (want[key] is None)
            if want[key] is not None:
                assert torch.equal(got[key].view(torch.int64), want[key].view(torch.int64)), "series differ"
        else:
            assert got[key] == want[key], key


@pytest.mark.parametrize("stream", ["packed", "certified", "no_procs"])
def test_back_to_back_builds_equal_fresh_builds(cuda, stream):
    from traceml_b200 import _abi

    lib = _abi.lib()
    certified = stream == "certified"

    def batch(n, seed, first_step):
        recs = pr._recs(n, seed, first_step=first_step)
        # certified: a wide record inside the window, so the pass streams the hot halves
        return pr._wide(recs, [n - 1000]) if certified else recs

    eng = _engine(procs=stream != "no_procs")
    try:
        summ = _summary(eng)
        steps = [("load", batch(250_000, 70, 1000)), (None, None),
                 ("commit", pr._recs(200, 71, first_step=1000 + 250_000)),
                 ("load", batch(260_000, 72, 1000 + 250_200)), (None, None),
                 ("reset", batch(240_000, 73, 17))]
        got, want = [], []
        for kind, recs in steps:
            if kind == "reset":
                eng.reset()
                kind = "load"
            if kind is not None:
                dc._apply(eng, [(kind, recs)])
            assert lib.tml_ring_certified_(eng.handle, W) == 1
            assert lib.tml_ring_packed_(eng.handle, W) == (0 if certified else 1)
            res = summ.build(W, PROCS)
            got.append((res, _facts(res)))
            want.append(_fresh(eng))  # a fresh engine, its text emitted on access
        # every build but the last had its text emitted by the build after it
        assert all(r._raw is not None for r, _ in got[:-1]) and got[-1][0]._raw is None
        for (res, facts), (wfacts, wtext) in zip(got, want):
            assert facts["fused_rows"] and facts["n_common"] == W
            _same(facts, wfacts)
            assert bytes(res.raw) == wtext
    finally:
        eng.close()


def test_kept_result_survives_later_builds(cuda):
    from traceml_b200 import _abi

    eng = _engine(procs=True)
    try:
        dc._apply(eng, [("load", pr._recs(250_000, 80))])
        summ = _summary(eng)
        kept = summ.build(W, PROCS)
        struct = bytes(kept["reduce"].out)
        timings = dict(kept["reduce"].timings_ms)
        # the text its struct gives, from a copy no build can touch
        text = _abi._sections_text(_abi.ReduceRunOut.from_buffer_copy(struct), kept._args)
        for i in range(3):
            dc._apply(eng, [("commit", pr._recs(50, 81 + i, first_step=1000 + 250_000 + 50 * i))])
            later = summ.build(W, PROCS)
            assert later["reduce"].out is not kept["reduce"].out
        assert bytes(kept["reduce"].out) == struct
        assert kept["reduce"].timings_ms == timings
        assert bytes(kept.raw) == text  # emitted by the build after it
        assert kept["step_time"]["data"]["aligned_window"]["end_step"] == 1000 + 250_000 - 1
    finally:
        eng.close()
