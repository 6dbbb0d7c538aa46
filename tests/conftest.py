"""pytest configuration: markers + import path.

``-m "not gpu"``: oracle vs golden vectors, host logic, C-ABI symbol checks,
world_size-2 gloo runs -- no CUDA device needed.
``-m gpu``: parity tests proper, through the C-ABI on a real H100.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_sessionstart(session):
    """Build the native library in-tree if it is missing (a fresh checkout has no .so: they
    are git-ignored).  nvcc cross-compiles without a GPU; after build() this is a no-op."""
    try:
        import __graft_entry__ as entry

        if not os.path.exists(entry.LIB):
            entry.build_native()
    except Exception as exc:  # the ABI tests then fail loudly with the real reason
        print(f"[conftest] native build skipped: {exc}", file=sys.stderr)
