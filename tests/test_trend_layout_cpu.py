"""CPU: ``reduce.trend_layout`` (the band index ranges K4b sums) against the oracle's trend evidence,
for every series length from 0 to 25 000 and both parameter sets.  The C++ ``trend_layout`` of the
native driver keeps the same arithmetic; ``test_gpu_align_bands.py::test_build_band_layout`` checks
it through a build."""
import math

import numpy as np
import pytest

from oracle import trend_oracle
from traceml_b200.reduce import trend_layout

PARAMS = [(200, 0.10), (50, 0.0)]
EDGES = sorted(set(range(199, 226)) | {49, 50, 51, 9_999, 10_000, 10_001, 11_111, 25_000})


def _oracle_layout(n, min_points, warm):
    """The index ranges trend_evidence averages over n points: its history cut and warm-up trim, then
    ``trend_oracle.band_bounds`` of the stable part, as global indices."""
    if n < min_points:
        return None
    length = min(n, 10_000)
    w = int(math.floor(length * warm))
    stable = length - w
    if stable < min_points:
        return None
    bands = (trend_oracle.BASELINE_BAND, trend_oracle.MID_BAND, trend_oracle.RECENT_BAND)
    return [tuple(n - length + w + e for e in trend_oracle.band_bounds(stable, b)) for b in bands]


@pytest.mark.parametrize("min_points,warm", PARAMS)
def test_trend_layout_every_length(min_points, warm):
    for n in range(0, 25_001):
        lay = trend_layout(n, min_points=min_points, warmup_frac=warm)
        exp = _oracle_layout(n, min_points, warm)
        assert (lay is None) == (exp is None), n
        if lay is not None:
            assert [tuple(b) for b in lay] == exp, n


@pytest.mark.parametrize("min_points,warm", PARAMS)
def test_oracle_layout_is_what_trend_evidence_averages(min_points, warm, monkeypatch):
    """The restatement above against trend_evidence itself: over a series whose values are their
    indices, the slices it averages are the band ranges."""
    seen = []
    mean = trend_oracle._mean
    monkeypatch.setattr(trend_oracle, "_mean", lambda v: (seen.append(list(v)), mean(v))[1])
    for n in EDGES + list(range(0, 1_200, 7)):
        seen.clear()
        ev = trend_oracle.trend_evidence([float(i) for i in range(n)], min_points=min_points, warmup_frac=warm)
        exp = _oracle_layout(n, min_points, warm)
        assert (ev is None) == (exp is None), n
        if ev is not None:
            assert [(int(v[0]), int(v[-1]) + 1) for v in seen] == exp, n
            assert all(np.array_equal(v, np.arange(v[0], v[-1] + 1)) for v in seen), n
