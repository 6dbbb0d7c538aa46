"""CPU side of the live layer-time panel: the numpy restatement of the reference's layer-time rules
pinned against the reference's own ``LayerCombinedTimerData`` on the seeded records,
``to_reference_layer_time`` driving the reference's layer-time renderer, and the C-ABI of the
device stages."""
import dataclasses
import io
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import layer_tick_cases as ltc  # noqa: E402


def _names(n):
    return [f"block.{i}.op" for i in range(n)]


@pytest.mark.parametrize("case", ltc.SEEDED)
@pytest.mark.parametrize("n_layers", [1, 33])
def test_restatement_matches_the_reference(monkeypatch, case, n_layers):
    if not ltc.reference_importable():
        pytest.skip("reference not installed in oracle/_ref")
    world, recs, ring = ltc.seeded(case, n_layers)
    recs = ltc.retained(recs, ring)
    names = _names(n_layers)
    ref = ltc.reference_computer(monkeypatch, world)
    got = ltc.reference_tick(ref, recs, names)
    ltc.check_first_tick(got, ltc.restate(recs, world), names, world)


def test_to_reference_layer_time_drives_the_kept_renderer(monkeypatch):
    if not ltc.reference_importable():
        pytest.skip("reference not installed in oracle/_ref")
    pytest.importorskip("rich")
    from rich.console import Console
    from traceml.renderers.layer_combined_time.renderer import LayerCombinedTimeRenderer

    from traceml_b200.reporting import ReferenceComputerAdapter, to_reference_layer_time

    world, recs, ring = ltc.seeded("missing_safe", 40)
    names = _names(40)

    class Dicts:  # a computer returning plain dicts, as live.LayerCombinedTimerData does
        def __init__(self):
            self.ref = ltc.reference_computer(monkeypatch, world, top_n_layers=5)

        def compute_display_data(self):
            return ltc.reference_tick(self.ref, recs, names)

    def text(renderer):
        c = Console(width=200, record=True, file=io.StringIO(), color_system=None)
        c.print(renderer.get_panel_renderable())
        return c.export_text()

    want = LayerCombinedTimeRenderer(top_n_layers=5, remote_store=ltc.reference_store(recs, names))
    want._service = ltc.reference_computer(monkeypatch, world, top_n_layers=5)
    want._service._remote_store = ltc.reference_store(recs, names)
    ours = LayerCombinedTimeRenderer(top_n_layers=5)
    ours._service = ReferenceComputerAdapter(Dicts(), to_reference_layer_time)
    a, b = text(ours), text(want)
    assert "missing ranks: [2]" in b and "Other Layers" in b
    assert a == b
    d = ours.get_dashboard_renderable()
    assert dataclasses.asdict(d)["safe_step"] == 9 and d.world_size == world


def test_layer_tick_abi():
    import ctypes as C

    from traceml_b200 import _abi

    lib = _abi.lib()
    for name in ("tml_layer_tick_bounds", "tml_layer_tick_snapshot", "tml_layer_tick_fold", "tml_layer_load_"):
        assert hasattr(lib, name) and name in _abi.SIGNATURES
    assert lib.tml_struct_size(b"tml_layer_snap") == C.sizeof(_abi.LayerSnap) == 48
    assert lib.tml_struct_size(b"tml_layer_tick_row") == C.sizeof(_abi.LayerTickRow) == 56
    from traceml_b200.live import _LAYER_ROW_DTYPE

    assert _LAYER_ROW_DTYPE.itemsize == C.sizeof(_abi.LayerTickRow)
    for f in ("cur_rank", "peak_rank", "peak_last", "worst_rank", "flags"):
        assert _LAYER_ROW_DTYPE.fields[f][1] == getattr(_abi.LayerTickRow, f).offset
    assert _LAYER_ROW_DTYPE.fields["cur_ms"][1] == _abi.LayerTickRow.cur_fwd_ms.offset
    assert _LAYER_ROW_DTYPE.fields["peak_ms"][1] == _abi.LayerTickRow.peak_fwd_ms.offset
    # without a layer ring the stages refuse, they do not guess
    assert lib.tml_layer_tick_snapshot(None, 0, None, None) < 0
    assert lib.tml_layer_tick_fold(None, None, 0, 0, None, None) < 0
