#!/usr/bin/env python
"""Pin oracle/timer_oracle.py against the reference's own timer path on CPU.

Runs the SAME scripted training loop (fake deterministic clock) through
  (1) the unmodified reference: traceml.utils.timing.timed_region,
      traceml.sdk.instrumentation.trace_step, StepTimeSampler / StepMemorySampler;
  (2) oracle.timer_oracle.ReferenceTimerPath
and asserts the emitted wire rows are identical; writes them to
tests/golden/timer_rows.json.  CPU only, so
this pins the host-clock half: step numbering, accumulate-by-name, n_calls,
dataloader_next flushed with the following step, failed-step flush under the
old id, NULL memory on CPU.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

import time  # noqa: E402

import torch  # noqa: E402


class FakeClock:
    def __init__(self):
        self.t = 1_700_000_000.0

    def __call__(self):
        self.t += 0.0005  # every read advances 0.5 ms -> deterministic durations
        return self.t


def script(timed_region, trace_step, model):
    """5 good steps + 1 failing step + 1 good step."""
    for i in range(7):
        with timed_region("_traceml_internal:dataloader_next", scope="step", use_gpu=False):
            pass
        try:
            with trace_step(model):
                for _ in range(2):
                    with timed_region("_traceml_internal:h2d_time", scope="step", use_gpu=True):
                        pass
                with timed_region("_traceml_internal:forward_time", scope="step", use_gpu=True):
                    pass
                if i == 5:
                    raise ValueError("boom")
                with timed_region("_traceml_internal:backward_time", scope="step", use_gpu=True):
                    pass
                with timed_region("_traceml_internal:optimizer_step", scope="step", use_gpu=True):
                    pass
        except ValueError:
            pass


def run_reference():
    import traceml.utils.timing as rt
    from traceml.runtime.state import reset_trace_session_state
    from traceml.samplers.step_memory_sampler import StepMemorySampler
    from traceml.samplers.step_time_sampler import StepTimeSampler
    from traceml.sdk.instrumentation import trace_step

    reset_trace_session_state(0)
    clock = FakeClock()
    real = time.time
    time.time = clock
    try:
        model = torch.nn.Linear(2, 2)
        script(rt.timed_region, trace_step, model)
        ts, ms = StepTimeSampler(), StepMemorySampler()
        ts.sample()
        ms.sample()
    finally:
        time.time = real
    trows = [dict(r) for r in ts.db.get_table("StepTimeTable")]
    mrows = [dict(r) for r in ms.db.get_table("step_memory")]
    return trows, mrows


def run_oracle():
    from oracle.timer_oracle import ReferenceTimerPath

    ref = ReferenceTimerPath()
    clock = FakeClock()
    real = time.time
    time.time = clock
    try:
        model = torch.nn.Linear(2, 2)
        script(ref.timed_region, ref.trace_step, model)
        out = ref.sample()
    finally:
        time.time = real
    return out["step_time"], out["step_memory"]


def norm(rows, drop=("seq", "ts", "model_id")):
    return [{k: v for k, v in r.items() if k not in drop} for r in rows]


def main():
    rt_rows, rm_rows = run_reference()
    ot_rows, om_rows = run_oracle()
    a, b = norm(rt_rows), norm(ot_rows)
    assert len(a) == len(b) == 7, (len(a), len(b))
    for x, y in zip(a, b):
        assert x["step"] == y["step"], (x["step"], y["step"])
        assert set(x["events"]) == set(y["events"])
        for name in x["events"]:
            for dev in x["events"][name]:
                ex, ey = x["events"][name][dev], y["events"][name][dev]
                assert ex["n_calls"] == ey["n_calls"] and ex["is_gpu"] == ey["is_gpu"]
                assert abs(ex["duration_ms"] - ey["duration_ms"]) < 1e-6, (name, ex, ey)
    assert norm(rm_rows) == norm(om_rows), (rm_rows, om_rows)
    with open(os.path.join(HERE, "timer_rows.json"), "w") as fh:
        json.dump({"step_time": norm(rt_rows), "step_memory": norm(rm_rows),
                   "steps": [r["step"] for r in rt_rows]}, fh, indent=1, sort_keys=True)
    print("timer oracle pinned; steps:", [r["step"] for r in rt_rows])
    print(json.dumps(norm(rt_rows)[5], indent=0)[:400])


if __name__ == "__main__":
    main()
