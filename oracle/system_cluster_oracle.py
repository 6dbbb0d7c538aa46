"""Oracle: the System section over several nodes.  TEST INFRASTRUCTURE ONLY.

Restates ``src/traceml/reporting/sections/system/loader.py:170-193,300-359`` for a run whose
System rows come from several sources (one per node leader), on top of the one-node restatement
in ``system_oracle``:
  - the window is the latest ``max_rows`` samples of each node, partitioned by
    ``COALESCE(node_rank, global_rank, 0)``;
  - the cluster aggregate runs over all retained rows ordered by that key (as an integer), then
    by insertion order;
  - ``nodes`` is keyed by the node label and built in the string order of the labels;
  - ``expected_nodes``: the one ``ceil(world_size / local_world_size)`` all rows agree on, else
    the number of distinct labels (loader.py:159-167);
  - the diagnosis is ``system_oracle.diagnose`` over those nodes (api.py:189-209).
Each source must carry its own node label (the product keeps one source per label).
"""

from __future__ import annotations

import math
from typing import Any, Dict, List, Sequence

from .system_oracle import aggregate, diagnose, per_gpu


def _label(identity: Dict[str, Any]) -> str:  # loader.py:78-81
    if identity.get("node_rank") is not None:
        return str(int(identity["node_rank"]))
    return str(int(identity.get("global_rank") or 0))


def _key(identity: Dict[str, Any]) -> int:  # COALESCE(node_rank, global_rank, 0)
    if identity.get("node_rank") is not None:
        return int(identity["node_rank"])
    return int(identity.get("global_rank") or 0)


def cluster_section(rows_by_node: Sequence[List[Dict[str, Any]]], identities: Sequence[Dict[str, Any]],
                    max_rows: int) -> Dict[str, Any]:
    """``rows_by_node[k]``: the wire rows of source k in insertion order, ``identities[k]`` its
    sampler identity.  Returns the dict ``traceml_b200.sections.build_system_cluster`` returns."""
    labels = [_label(i) for i in identities]
    assert len(set(labels)) == len(labels), "one source per node label"
    wins = [list(rows)[-int(max_rows):] if max_rows > 0 else [] for rows in rows_by_node]
    order = sorted(range(len(wins)), key=lambda k: _key(identities[k]))
    concat = [r for k in order for r in wins[k]]
    nodes: Dict[str, Any] = {}
    for k in sorted(range(len(wins)), key=lambda k: labels[k]):
        if not wins[k]:
            continue
        ident = {"label": labels[k]}
        ident.update({f: identities[k].get(f) for f in ("node_rank", "hostname", "global_rank", "local_rank",
                                                        "local_world_size", "world_size")})
        nodes[labels[k]] = {"identity": ident, "aggregate": aggregate(wins[k]), "per_gpu": per_gpu(wins[k])}
    present = [identities[k] for k in range(len(wins)) if wins[k]]
    cands = {int(math.ceil(float(i["world_size"]) / float(i["local_world_size"])))
             for i in present if i.get("world_size") and i.get("local_world_size")}
    expected = max(1, cands.pop()) if len(cands) == 1 else max(1, len({_label(i) for i in present}))
    agg = aggregate(concat)
    return {"aggregate": agg, "nodes": nodes, "expected_nodes": expected, "diagnosis": diagnose(agg, nodes)}
