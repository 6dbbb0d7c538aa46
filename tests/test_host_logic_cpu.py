"""CPU: host-side logic of the reduce (band layout, info packing, rollups)."""
import math
import random

import numpy as np
import pytest

from oracle import step_time_oracle, trend_oracle
from traceml_b200.reduce import WindowReducer, trend_layout


@pytest.mark.parametrize("min_points,warm", [(200, 0.10), (50, 0.0)])
def test_trend_layout_matches_reference_bands(min_points, warm):
    rng = np.random.default_rng(0)
    for n in [1, 49, 50, 51, 199, 200, 201, 222, 223, 260, 999, 1000, 1001, 9_999, 10_000, 10_001, 25_017]:
        series = rng.uniform(1.0, 2.0, n).tolist()
        ev = trend_oracle.trend_evidence(series, min_points=min_points, warmup_frac=warm)
        lay = trend_layout(n, min_points=min_points, warmup_frac=warm)
        assert (ev is None) == (lay is None), n
        if ev is None:
            continue
        a = np.asarray(series)
        for (lo, hi), key in zip(lay, ("baseline_avg", "mid_avg", "recent_avg")):
            assert math.isclose(a[lo:hi].sum() / (hi - lo), ev[key], rel_tol=1e-13), (n, key)


def test_win_info_pack_roundtrip():
    """A rank's ``WinInfo`` through the exchange layout and back into a ``WinInfo``, with the
    memory candidate bounds it advertises."""
    from traceml_b200 import _abi

    w = _abi.WinInfo(n_retained=12345, latest_step=2 ** 40 + 7, monotone=1, dup_rows=3, n_rows=(100, 200),
                     n_cand=(99, 198), lo=(5, 6), hi=(2 ** 40, 2 ** 40 + 7),
                     t_sums=(1.5, 2.5, 3.5, 4.5, 5.5, 6.5, 7.5), t_count=99, n_both=98, dense=(1, 0))
    v = WindowReducer._info_pack(w, (w.lo[1], w.n_cand[1]))
    assert len(v) == 23
    got = _abi.WinInfo()
    WindowReducer._info_unpack([float(x) for x in v], got)
    assert bytes(got) == bytes(w)
    WindowReducer._info_unpack([float(x) for x in WindowReducer._info_pack(w, (2 ** 40 - 3, 4))], got)
    assert (got.lo[1], got.n_cand[1]) == (2 ** 40 - 3, 4)  # the advertised memory candidates
    assert (got.lo[0], got.n_cand[0], got.hi[1]) == (5, 99, 2 ** 40 + 7)


def _step_time_of_sums(sums_by_rank, n):
    """The Step-Time section tml_sections_json emits for a reduce whose aligned window holds ``n``
    steps of every rank in ``sums_by_rank`` with these seven per-metric sums."""
    from traceml_b200 import _abi

    o = _abi.ReduceRunOut()
    o.n_ranks = max(1, len(sums_by_rank))
    k = o.time
    k.observed = k.n_used = len(sums_by_rank)
    k.n_common = n
    for i, (r, s) in enumerate(sorted(sums_by_rank.items())):
        k.used[i], k.n_rows[i] = r, n
        k.t_sums[i][:] = s
    return _abi.sections_json(o, 1.0e9, 1, 10_000, 0)["step_time"]


def test_emitted_rollups_match_oracle_on_random_ranks():
    rnd = random.Random(3)
    for R in (1, 2, 3, 4, 7, 8):
        n = rnd.randint(1, 500)
        sums = {}
        for r in range(R):
            f, b, o = rnd.uniform(5, 15) * n, rnd.uniform(10, 30) * n, rnd.uniform(1, 5) * n
            traced = f + b + o + rnd.uniform(0, 10) * n
            dl = rnd.uniform(1, 50) * n
            sums[r] = [dl, f, b, o, traced, traced, dl + traced]
        got = _step_time_of_sums(sums, n)
        summ = {r: step_time_oracle._summary(n, *s) for r, s in sums.items()}
        assert got["global"] == step_time_oracle.global_points(summ)
        assert got["overview"] == step_time_oracle.overview(summ)
    none = _step_time_of_sums({}, 0)["overview"]
    assert none["rank_comparison"] == "no_data" and none == step_time_oracle.overview({})


def test_b_reduce_formula():
    import importlib.util
    import os

    spec = importlib.util.spec_from_file_location(
        "bench", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    assert bench.b_reduce(8, 10_000) == 8 * 10_000 * 64 + 128 * 10_000 + 72 * 8  # SURVEY 8d: ~6.4 MB


def test_summary_artifacts_are_written_atomically(tmp_path):
    """final_summary.json / .txt: names and format of sdk/protocol.py:160-171, atomic replace."""
    import json

    from traceml_b200.summary import write_summary_artifacts

    env = {"schema_version": "1.2", "step_time": {"x": 1.5}, "text": "Step Time: BALANCED"}
    paths = write_summary_artifacts(env, str(tmp_path / "session"))
    assert json.load(open(paths["json"])) == env
    assert open(paths["json"]).read() == json.dumps(env, indent=2)
    assert open(paths["txt"]).read() == "Step Time: BALANCED"
    write_summary_artifacts(dict(env, text="again"), str(tmp_path / "session"))  # replace in place
    assert open(paths["txt"]).read() == "again"
    assert sorted(p.name for p in (tmp_path / "session").iterdir()) == ["final_summary.json", "final_summary.txt"]


def test_auto_exchange_avoids_p2p_across_hosts():
    """``auto`` picks the CUDA-IPC peer-load exchange from 10^6 aligned rows per rank -- only when
    every rank is a process of this host (reduce.py:_exchange_mode, run_native)."""
    import torch
    from fake_engine import FakeEngine
    import replay
    from traceml_b200.reduce import WindowReducer

    class Comm:
        world, index = 2, 0

        def __init__(self, same):
            self.same, self.asked = same, 0

        def one_host(self, device=None):
            self.asked += 1
            return self.same

    eng = FakeEngine(replay.make_step_replay("balanced", 1, 8, seed=0)[0], None)
    for same, big in ((True, "p2p"), (False, "a2a")):
        red = WindowReducer([eng], Comm(same), device=torch.device("cuda", 0), exchange="auto")
        assert red._exchange_mode(10_000) == "a2a"            # small windows never map peers
        assert red._exchange_mode(2_000_000) == big
        assert red._spec_len() == (15 + 72 if same else 15)   # no IPC handle in the first exchange
    red = WindowReducer([eng], Comm(False), device=torch.device("cuda", 0), exchange="p2p")
    assert red._exchange_mode(2_000_000) == "p2p"             # an explicit request is honoured
    # a communicator object without the method (user-supplied): assume one host, as before
    class Bare:
        world, index = 2, 0
    assert WindowReducer([eng], Bare(), device=torch.device("cuda", 0))._exchange_mode(2_000_000) == "p2p"
