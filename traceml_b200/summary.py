"""``final_summary()`` -- in-process end-of-run summary.

The reference answers ``traceml.final_summary()`` with a file request/response
round trip to the aggregator process, which runs the sections over SQLite
(``src/traceml/sdk/summary_client.py:35``, ``aggregator/summary_service.py:27-114``).
Here every rank already holds its window in HBM, so the summary is one
collective call: all ranks enter, rank 0 (or every rank) gets the result.
"""
from __future__ import annotations

import json
import os
from typing import Any, Dict, Optional

from .runtime import disabled, get_engine, summary_window_rows


def _replace_with(path: str, text: str) -> None:
    """Readers never see a half-written artifact: sibling temp file, fsync, rename."""
    folder = os.path.dirname(os.path.abspath(path))
    os.makedirs(folder, exist_ok=True)
    tmp = os.path.join(folder, f".{os.path.basename(path)}.{os.getpid()}.tmp")
    try:
        with open(tmp, "w", encoding="utf-8") as fh:
            fh.write(text)
            fh.flush()
            os.fsync(fh.fileno())
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)


def write_summary_artifacts(summary: Dict[str, Any], session_root: str) -> Dict[str, str]:
    """``<session>/final_summary.json`` (``json.dumps(indent=2)``) and ``final_summary.txt``:
    the artifact names and format of ``sdk/protocol.py:160-171`` / ``utils/atomic_io.py:18-63``
    that ``traceml compare`` and the launcher's end-of-run printout read."""
    root = os.path.abspath(session_root)
    paths = {"json": os.path.join(root, "final_summary.json"), "txt": os.path.join(root, "final_summary.txt")}
    _replace_with(paths["json"], json.dumps(summary, indent=2))
    _replace_with(paths["txt"], str(summary.get("text", "")))
    return paths


_CALLS = 0
MAX_RANKS = 64  # TML_MAX_RANKS (include/traceml_b200.h): ranks one reduce can align


def _rendezvous(timeout_sec: float, poll_interval_sec: float) -> bool:
    """All ranks have entered ``final_summary`` -- or nobody proceeds.

    The reference's call is a file RPC that any rank may issue alone and that returns ``None``
    after ``timeout_sec`` (``sdk/summary_client.py:35-110``).  Here the summary is a collective,
    so the time-out is honoured in front of it: ranks count themselves in through the process
    group's store and poll every ``poll_interval_sec``; the first rank to see everyone present
    publishes "go", the first to run out of time publishes "abort" (compare-and-set, so the
    decision is unanimous) and every rank returns ``None`` -- fail open, nothing hangs.
    """
    import time

    import torch.distributed as dist

    global _CALLS
    _CALLS += 1
    try:
        store = dist.distributed_c10d._get_default_store()
    except Exception:
        return True  # no store to meet on: enter the collective directly
    world = dist.get_world_size()
    key_n, key_d = f"traceml_b200/final_summary/{_CALLS}/n", f"traceml_b200/final_summary/{_CALLS}/d"
    deadline = time.monotonic() + max(0.0, float(timeout_sec))
    try:
        store.add(key_n, 1)
        while True:
            if store.add(key_n, 0) >= world:
                return store.compare_set(key_d, "", "go") == b"go"
            try:
                decided = store.compare_set(key_d, "", "")  # read without deciding
            except Exception:
                decided = b""
            if decided in (b"go", b"abort"):
                return decided == b"go"
            if time.monotonic() >= deadline:
                return store.compare_set(key_d, "", "abort") == b"go"
            time.sleep(max(1e-3, float(poll_interval_sec)))
    except Exception as exc:
        import sys

        print(f"[TraceML] final_summary rendezvous failed ({exc}); entering the reduce directly", file=sys.stderr)
        return True


def final_summary(*, timeout_sec: float = 30.0, poll_interval_sec: float = 0.1,
                  print_text: bool = False, rank0_only: bool = True,
                  window_rows: Optional[int] = None,
                  session_root: Optional[str] = None) -> Optional[Dict[str, Any]]:
    """Collective over the default process group when one is initialised; ``timeout_sec`` /
    ``poll_interval_sec`` bound the wait for the other ranks (``None`` is returned on every rank
    if one never arrives -- same fail-open contract as ``sdk/summary_client.py:35``).
    ``session_root`` (default: ``$TRACEML_SESSION_ROOT`` if set): where rank 0 also writes the
    artifacts."""
    if disabled():
        return None
    import torch
    import torch.distributed as dist

    from .reduce import LocalComm, TorchDistComm
    from .reporting import build_final_summary
    from .sections import SummaryEngine

    import sys

    distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    if distributed and dist.get_world_size() > MAX_RANKS:
        if dist.get_rank() == 0:
            print(f"[TraceML] final_summary: {dist.get_world_size()} ranks exceed the {MAX_RANKS} one "
                  "reduce aligns; no summary produced", file=sys.stderr)
        return None
    if distributed and not _rendezvous(timeout_sec, poll_interval_sec):
        print(f"[TraceML] final_summary: not every rank arrived within {timeout_sec:.1f} s; "
              "no summary produced", file=sys.stderr)
        return None
    eng = get_engine()
    # every stream of the device, torch's internal NCCL stream included: the native reduce issues
    # its collectives on torch.distributed's own communicator, which must be idle by then (all ranks
    # are here -- the rendezvous -- so whatever they had in flight completes)
    torch.cuda.synchronize(torch.device("cuda", eng.device))
    comm = TorchDistComm() if distributed else LocalComm()
    res = SummaryEngine([eng], comm).build(window_rows or summary_window_rows(),
                                           window_rows or summary_window_rows())
    if rank0_only and comm.index != 0:
        return None
    if distributed and not rank0_only:
        # one System source (local rank 0 = comm index 0): every rank reports its section
        box = [res["system"] if comm.index == 0 else None]
        dist.broadcast_object_list(box, src=0)
        res["system"] = box[0]
    out = build_final_summary(res)
    root = session_root or os.environ.get("TRACEML_SESSION_ROOT")
    if root and comm.index == 0:
        try:
            write_summary_artifacts(out, root)
        except OSError as exc:  # artifacts are best effort; the caller still gets the summary
            import sys

            print(f"[TraceML] could not write final summary artifacts: {exc}", file=sys.stderr)
    if print_text and out.get("text"):
        print(out["text"])
    return out


__all__ = ["final_summary", "write_summary_artifacts"]
