"""CPU oracle for the traceml_b200 hot path.  TEST INFRASTRUCTURE ONLY.

This package is a plain-Python/numpy restatement of the arithmetic that the
reference (traceopt-ai/traceml @ a659c95, v0.2.15) performs on the telemetry
hot path: step alignment, per-rank / cross-rank step-time and step-memory
reduction, process aggregation, and the three rule engines that turn those
numbers into diagnosis labels.  Every function cites the reference file:line
it follows.

Rules of use (enforced by tests/test_abi_cpu.py):
  * only ``tests/``, ``__graft_entry__.smoke()``, ``bench.py``'s
    ``cpu_baseline`` / ``--impl reference`` legs and ``__graft_entry__.build()`` (for
    ``oracle/install_reference.py``, which installs the reference) may import this package;
  * nothing under ``traceml_b200/`` imports it -- the product path is the CUDA
    extension and fails loudly when that is missing.

Parity pin: ``oracle/`` is checked against the reference itself, installed in
``oracle/_ref`` (oracle/install_reference.py), by
``tests/golden/make_golden.py`` (final-summary sections, 33 cases),
``make_live_golden.py`` (live views, 26 cases), ``make_fuzz_golden.py`` (seeded random
cases) and ``make_timer_golden.py`` (timer path); the
resulting vectors (inputs + the reference's own outputs) are committed under
``tests/golden/`` and re-checked on every CPU test run (tests/test_oracle_golden.py,
tests/test_live_cpu.py, tests/test_timer_oracle_cpu.py).
"""
