"""GPU: the UNMODIFIED reference's public API (``import traceml``; init / trace_step, its own
patches and step counter) recording through this engine's C-ABI via traceml_b200.shim.

Runs in a fresh interpreter: the reference and this package mark their monkey patches with the
same attribute names (``torch.Tensor._traceml_h2d_patched`` ...), so in a process where this
package's own ``init`` already ran the reference would -- correctly -- refuse to patch again.  In
an option-B deployment only the reference's ``init`` runs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

SCRIPT = r"""
import os, sys
ROOT, REF = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT); sys.path.insert(0, REF)
os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
import torch
torch.cuda.set_device(0)
import traceml                                   # the reference
from traceml.runtime.state import reset_trace_session_state
from traceml_b200 import runtime, shim

assert "oracle/_ref" in traceml.__file__.replace(os.sep, "/")
patched = shim.install()
assert "traceml.sdk.instrumentation.timed_region" in patched
reset_trace_session_state(0)
traceml.init(mode="auto")                        # the reference's own init: ITS patches
eng = runtime.get_engine()
torch.cuda.synchronize(); eng.drain()
model = torch.nn.Sequential(torch.nn.Linear(128, 256), torch.nn.ReLU(), torch.nn.Linear(256, 8)).cuda()
opt = torch.optim.SGD(model.parameters(), lr=0.01)
ds = torch.utils.data.TensorDataset(torch.randn(32 * 5, 128), torch.randint(0, 8, (32 * 5,)))
expect = []
for x, y in torch.utils.data.DataLoader(ds, batch_size=32):
    with traceml.trace_step(model):              # the reference's own context manager
        x, y = x.to("cuda"), y.to("cuda")
        loss = torch.nn.functional.cross_entropy(model(x), y)
        loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)
        expect.append(torch.cuda.max_memory_allocated(0))
torch.cuda.synchronize()
recs, dropped = eng.drain()
assert dropped == 0 and list(recs["step"]) == [1, 2, 3, 4, 5], list(recs["step"])   # its step counter
assert (recs["n_calls"][:, 0] == 1).all(), recs["n_calls"][:, 0]      # dataloader_next (its patch)
assert (recs["n_calls"][:, 1] == 2).all(), recs["n_calls"][:, 1]      # two H2D copies (its patch)
assert (recs["n_calls"][:, 2:6] == 1).all() and (recs["dur_ns"][:, 2:6] > 0).all(), (recs["n_calls"], recs["dur_ns"])
assert (recs["gpu_mask"] == 0b011110).all()                            # device-stamped phases
assert [int(v) for v in recs["peak_alloc"]] == expect                  # a5 through the shim
from traceml.samplers.step_time_sampler import StepTimeSampler       # rebound to the ring drain
with traceml.trace_step(model):
    model(torch.randn(4, 128, device="cuda")).sum().backward()
torch.cuda.synchronize()
s = StepTimeSampler(); s.sample()
rows = list(s.db.all_tables()["StepTimeTable"])
assert len(rows) == 1 and rows[0]["step"] == 6 and "_traceml_internal:forward_time" in rows[0]["events"]
shim.uninstall()
print("SHIM_OK", len(patched))
"""


def test_reference_trace_step_records_through_the_c_abi():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if not os.path.isdir(os.path.join(REF, "traceml")):
        pytest.skip("oracle/_ref (the installed reference) is not present")
    p = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, REF], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "SHIM_OK" in p.stdout, (p.stdout[-2000:], p.stderr[-3000:])
