"""The KEPT live renderers fed from this package (SURVEY 8b down-facing seam, 8f-2): the
reference's own ``StepCombinedRenderer`` / ``StepMemoryRenderer`` render the same panel text
whether their computer reads the reference's SQLite (the reference path) or is replaced by
``traceml_b200.live`` over the engine double.  Needs the reference installed in oracle/_ref."""
import io
import os
import sys
import tempfile

import pytest
import torch

REF_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
if os.path.isdir(REF_SRC) and REF_SRC not in sys.path:
    sys.path.insert(0, REF_SRC)
pytest.importorskip("traceml.renderers.step_time.renderer", reason="reference not importable here")
pytest.importorskip("rich")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


def _text(panel) -> str:
    from rich.console import Console

    c = Console(width=200, record=True, file=io.StringIO(), color_system=None)
    c.print(panel)
    return c.export_text()


@pytest.mark.parametrize("scenario,R,S,seed", [("input_straggler", 4, 460, 0), ("balanced", 1, 300, 13),
                                              ("ragged", 4, 300, 8), ("mem_imbalance", 4, 260, 18),
                                              ("wait_heavy", 8, 260, 5)])
def test_kept_renderers_render_identically(scenario, R, S, seed):
    import make_golden as mg
    from fake_engine import FakeEngine
    from traceml.renderers.step_memory.renderer import StepMemoryRenderer
    from traceml.renderers.step_time.renderer import StepCombinedRenderer
    import replay
    from traceml_b200.live import StepCombinedComputer, StepMemoryMetricsComputer
    from traceml_b200.reporting import (ReferenceComputerAdapter, to_reference_step_combined,
                                        to_reference_step_memory_combined)

    recs = replay.make_step_replay(scenario, R, S, seed)
    engines = [FakeEngine(recs[r]) for r in sorted(recs)]
    cpu = torch.device("cpu")
    with tempfile.TemporaryDirectory() as td:
        db = os.path.join(td, "telemetry")
        mg.build_db(db, step_records=recs)
        ref_t, ref_m = StepCombinedRenderer(db), StepMemoryRenderer(db)
        want_t, want_m = _text(ref_t.get_panel_renderable()), _text(ref_m.get_panel_renderable())
        ours_t, ours_m = StepCombinedRenderer(db), StepMemoryRenderer(db)
        ours_t._computer = ReferenceComputerAdapter(StepCombinedComputer(engines, device=cpu),
                                                    to_reference_step_combined)
        ours_m._computer = ReferenceComputerAdapter(
            StepMemoryMetricsComputer(engines, device=cpu, gpu_available=None),
            to_reference_step_memory_combined)
        got_t, got_m = _text(ours_t.get_panel_renderable()), _text(ours_m.get_panel_renderable())
        # dashboard payloads: the typed objects themselves
        assert ours_t.get_dashboard_renderable().rank_heatmap == ref_t.get_dashboard_renderable().rank_heatmap
    assert "Waiting for first" not in want_t
    assert got_t == want_t
    # the memory panel prints the majority device label, a Python-set tie-break in the reference
    # (common.py:400-408): compare with the label column neutralised
    import re

    strip = lambda s: re.sub(r"cuda:\\d+|—", "", s)  # noqa: E731
    assert strip(got_m).split() == strip(want_m).split()
