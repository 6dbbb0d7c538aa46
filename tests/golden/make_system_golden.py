"""Generate tests/golden/system/*.json from the UNMODIFIED reference (needs oracle/_ref).

Each seeded sample stream (tests/system_cases.py) goes through the reference's own SQLite writer
(aggregator/sqlite_writers/system.py ``init_schema`` / ``build_rows`` / ``insert_rows``), then
``SystemSummarySection(max_system_rows=W).build(db)``.  The golden keeps the loaded section data,
the diagnosis, the payload and the card text; the generator asserts that oracle/system_oracle.py
reproduces the data and the diagnosis with ``==`` before it writes anything.  The sha256 of the
input wire rows is pinned, as make_golden.py does for its replays.

    python tests/golden/make_system_golden.py
"""
from __future__ import annotations

import dataclasses
import hashlib
import json
import os
import sqlite3
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
os.environ.setdefault("TRACEML_LOGS_DIR", os.path.join(tempfile.gettempdir(), "traceml_ref_logs"))

import system_cases as sc  # noqa: E402
from oracle import system_oracle  # noqa: E402


def wire_digest(rows) -> str:
    return hashlib.sha256(json.dumps(rows, sort_keys=True).encode()).hexdigest()


def build_db(path: str, rows, identity) -> None:
    """The node's wire rows through the reference's writer, one sampler payload per row
    (SystemSampler flushes one row per send: runtime/sampler_registry.py:78-105)."""
    from traceml.aggregator.sqlite_writers import system as w

    conn = sqlite3.connect(path)
    w.init_schema(conn)
    for i, row in enumerate(rows):
        payload = dict(identity, rank=identity["global_rank"], sampler="SystemSampler", timestamp=row["ts"],
                       tables={"SystemTable": [row]})
        w.insert_rows(conn, w.build_rows(payload, recv_ts_ns=i + 1))
    conn.commit()
    conn.close()


def _plain(x):
    if dataclasses.is_dataclass(x):
        return {f.name: _plain(getattr(x, f.name)) for f in dataclasses.fields(x)}
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


def reference_section(db: str, window: int):
    from traceml.reporting.sections.system import SystemSummarySection

    sec = SystemSummarySection(max_system_rows=window)
    data = sec.load(db)
    diag = sec.diagnose(sec.to_diagnosis_input(data))
    res = sec.build_payload(data, diag)
    c = data.cluster
    section = {"aggregate": _plain(c.aggregate),
               "nodes": {label: {"identity": _plain(n.identity), "aggregate": _plain(n.aggregate),
                                 "per_gpu": {int(i): _plain(g) for i, g in n.per_gpu.items()}}
                         for label, n in c.nodes.items()},
               "expected_nodes": c.expected_nodes,
               "diagnosis": {"primary": _plain(diag.primary), "issues": _plain(list(diag.issues))}}
    for n in section["nodes"].values():
        for g in n["per_gpu"].values():
            g.pop("gpu_idx", None)
    return section, _plain(res.payload), res.text


def _comparable(section):
    """The oracle's section in the reference's shape (per-GPU rows without gpu_idx, issues as dicts)."""
    out = json.loads(json.dumps(section))
    for n in out["nodes"].values():
        n["per_gpu"] = {int(i): {k: v for k, v in g.items() if k != "gpu_idx"} for i, g in n["per_gpu"].items()}
    return out


def main() -> None:
    out_dir = os.path.join(HERE, "system")
    os.makedirs(out_dir, exist_ok=True)
    index = []
    for name, (G, n, window, _) in sc.CASES.items():
        raw = sc.make_raw(name)
        rows = [sc.wire_row(s) for s in raw]
        with tempfile.TemporaryDirectory() as td:
            db = os.path.join(td, "telemetry")
            build_db(db, rows, sc.IDENTITY)
            ref, payload, text = reference_section(db, window)
        mine = _comparable(system_oracle.system_section(rows, sc.IDENTITY, window))
        ref_cmp = json.loads(json.dumps(ref))
        ref_cmp["nodes"] = {k: dict(v, per_gpu={int(i): g for i, g in v["per_gpu"].items()})
                            for k, v in ref_cmp["nodes"].items()}
        assert mine == ref_cmp, (name, mine, ref_cmp)
        doc = {"case": name, "gpus": G, "samples": n, "window": window, "identity": sc.IDENTITY,
               "input_sha256": wire_digest(rows), "section": ref, "payload": payload, "text": text}
        with open(os.path.join(out_dir, f"{name}.json"), "w") as fh:
            json.dump(doc, fh, indent=1, sort_keys=True)
        index.append({"case": name, "kind": ref["diagnosis"]["primary"]["kind"],
                      "issues": [i["kind"] for i in ref["diagnosis"]["issues"]]})
    with open(os.path.join(out_dir, "INDEX.json"), "w") as fh:
        json.dump({"cases": index, "reference": "traceopt-ai/traceml v0.2.15 @ a659c95"}, fh, indent=1)
    print(f"wrote {len(index)} system golden cases")


if __name__ == "__main__":
    main()
