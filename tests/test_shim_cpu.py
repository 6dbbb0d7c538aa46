"""Option B shim (traceml_b200/shim.py): the reference package's seam is rebound in place, and
restored.  CPU: only the binding is checked (no region is entered); the GPU test runs the
reference's own trace_step through it (tests/test_gpu_shim.py)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CANDIDATES = [os.path.join(ROOT, "oracle", "_ref")]


@pytest.fixture()
def reference():
    path = next((p for p in CANDIDATES if os.path.isdir(os.path.join(p, "traceml"))), None)
    if path is None:
        pytest.skip("the reference package is not available")
    os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
    sys.path.insert(0, path)
    yield path
    sys.path.remove(path)


def test_install_rebinds_every_holder_and_uninstall_restores(reference):
    from traceml_b200 import shim
    from traceml_b200.utils import timing as mine_tm

    import traceml.sdk.instrumentation as ref_sdk
    import traceml.utils.timing as ref_tm

    orig_region = ref_tm.timed_region
    orig_flush = ref_sdk.flush_step_events
    patched = shim.install()
    try:
        assert shim.installed()
        assert ref_tm.timed_region is mine_tm.timed_region
        assert ref_sdk.timed_region is mine_tm.timed_region            # bound by `from ... import`
        assert ref_sdk.flush_step_events is not orig_flush
        import traceml.instrumentation.patches.forward_auto_timer_patch as fwd

        assert fwd.timed_region is mine_tm.timed_region
        for name in ("traceml.utils.timing.timed_region", "traceml.sdk.instrumentation.StepMemoryTracker",
                     "traceml.utils.flush_buffers.flush_step_events",
                     "traceml.samplers.step_time_sampler.StepTimeSampler"):
            assert name in patched, (name, patched)
        assert shim.install() == []                                       # idempotent
    finally:
        shim.uninstall()
    assert ref_tm.timed_region is orig_region and ref_sdk.flush_step_events is orig_flush
    assert not shim.installed()
