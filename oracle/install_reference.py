"""Install the unmodified reference package (traceopt-ai/traceml) into the git-ignored ``oracle/_ref``.

The reference is pure Python; ``pip install --target`` from a source tree is the whole recipe.
``bench.py --impl reference``, ``baseline/reference_legs.py`` and the tests that run the
reference's own code beside this package's read it from there.  The source tree is
``TRACEML_REFERENCE_SRC`` if set, else the reference checkout's default location
(``DEFAULT_SRC``); where neither holds one, nothing is installed and those consumers fall back
(bench) or skip (tests).  The comparisons that need only the reference's outputs do not depend on
it: they read golden vectors stored under ``tests/golden/``.

    python oracle/install_reference.py [SOURCE_TREE]
"""
from __future__ import annotations

import os
import shutil
import stat
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
DEFAULT_SRC = "/root/reference"  # traceopt-ai/traceml @ a659c95, read-only


def install(src: str | None = None, dst: str = DEST) -> bool:
    """True when ``dst`` holds an importable ``traceml`` package afterwards."""
    if os.path.isdir(os.path.join(dst, "traceml")):
        return True
    src = src or os.environ.get("TRACEML_REFERENCE_SRC") or DEFAULT_SRC
    if not os.path.isfile(os.path.join(src, "pyproject.toml")):
        return False
    with tempfile.TemporaryDirectory(prefix="tml_ref_") as tmp:
        work = os.path.join(tmp, "reference")  # build from a copy: the source tree may be read-only
        shutil.copytree(src, work, symlinks=True, ignore=shutil.ignore_patterns(".git"))
        for d, _, files in os.walk(work):  # the copy keeps read-only modes; the build writes into it
            for path in [d] + [os.path.join(d, f) for f in files]:
                if not os.path.islink(path):
                    os.chmod(path, os.stat(path).st_mode | stat.S_IWUSR)
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--target", dst, "-q", work]
        rc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if rc.returncode != 0:
        print(f"[oracle] reference not installed into {dst}: {rc.stdout[-400:]}", file=sys.stderr)
        return False
    return True


if __name__ == "__main__":
    sys.exit(0 if install(sys.argv[1] if len(sys.argv) > 1 else None) else 1)
