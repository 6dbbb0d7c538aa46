"""Generate tests/golden/system_cluster/*.json from the UNMODIFIED reference (needs oracle/_ref).

Each node's seeded sample stream (tests/system_cluster_cases.py) goes through the reference's own
SQLite writer with that node's identity, all nodes into one database, as make_system_golden.py
does for one node.  Then ``SystemSummarySection(max_system_rows=W).build(db)``.  The generator
asserts that oracle/system_cluster_oracle.py reproduces the data and the diagnosis with ``==``
before it writes anything; the sha256 of each node's wire rows is pinned.

    python tests/golden/make_system_cluster_golden.py
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
os.environ.setdefault("TRACEML_LOGS_DIR", os.path.join(tempfile.gettempdir(), "traceml_ref_logs"))

import make_system_golden as msg  # noqa: E402
import system_cases as sc  # noqa: E402
import system_cluster_cases as scc  # noqa: E402
from oracle import system_cluster_oracle  # noqa: E402


def main() -> None:
    out_dir = os.path.join(HERE, "system_cluster")
    os.makedirs(out_dir, exist_ok=True)
    index = []
    for name in scc.CASES:
        window, raws, idents = scc.make_case(name)
        rows = [[sc.wire_row(s) for s in raw] for raw in raws]
        with tempfile.TemporaryDirectory() as td:
            db = os.path.join(td, "telemetry")
            for node_rows, ident in zip(rows, idents):
                msg.build_db(db, node_rows, ident)
            ref, payload, text = msg.reference_section(db, window)
        mine = msg._comparable(system_cluster_oracle.cluster_section(rows, idents, window))
        ref_cmp = json.loads(json.dumps(ref))
        ref_cmp["nodes"] = {k: dict(v, per_gpu={int(i): g for i, g in v["per_gpu"].items()})
                            for k, v in ref_cmp["nodes"].items()}
        assert mine == ref_cmp, (name, mine, ref_cmp)
        doc = {"case": name, "window": window, "identities": idents,
               "samples": [len(r) for r in rows], "input_sha256": [msg.wire_digest(r) for r in rows],
               "section": ref, "payload": payload, "text": text}
        with open(os.path.join(out_dir, f"{name}.json"), "w") as fh:
            json.dump(doc, fh, indent=1, sort_keys=True)
        index.append({"case": name, "nodes": len(ref["nodes"]), "expected_nodes": ref["expected_nodes"],
                      "kind": ref["diagnosis"]["primary"]["kind"],
                      "issues": [i["kind"] for i in ref["diagnosis"]["issues"]]})
    with open(os.path.join(out_dir, "INDEX.json"), "w") as fh:
        json.dump({"cases": index, "reference": "traceopt-ai/traceml v0.2.15 @ a659c95"}, fh, indent=1)
    print(f"wrote {len(index)} system cluster golden cases")


if __name__ == "__main__":
    main()
