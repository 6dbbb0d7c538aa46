"""Seeded multi-node System streams (TEST INFRASTRUCTURE): one sample stream per node leader,
each a seeded stream of ``system_cases`` with its own launcher identity.  Shared by
``golden/make_system_cluster_golden.py`` and the cluster tests."""
from __future__ import annotations

import system_cases as sc

# name -> (window, [(base case of system_cases, seed, identity overrides), ...])
# Identities default to node k of a run of `nodes` x 8 GPUs (see identity()).
CASES = {
    "two_nodes_g8": (10_000, [("normal_g8", 0, {}), ("normal_g8", 1, {})]),
    "four_nodes_high_gpu_memory": (10_000, [("normal_g8", 0, {}), ("normal_g8", 1, {}),
                                            ("very_high_gpu_memory_g8", 2, {}), ("normal_g8", 3, {})]),
    "gpu_counts_8_4_1": (10_000, [("normal_g8", 0, {}), ("failed_gpu_g4", 1, {}), ("g1", 2, {})]),
    "cpu_only_node": (10_000, [("normal_g8", 0, {}), ("cpu_only", 1, {})]),
    "partial_coverage_3_of_4": (10_000, [("normal_g8", 0, {}), ("g3", 1, {}), ("no_data", 2, {}),
                                         ("normal_g8", 3, {})]),
    "eleven_nodes": (10_000, [(("g1", "g3", "normal_g8")[k % 3], k, {}) for k in range(11)]),
    "window_smaller": (64, [("window_smaller_g8", 0, {}), ("normal_g8", 1, {}), ("single_sample_g8", 2, {})]),
    "tie_broken_by_label": (10_000, [("high_cpu_g8", 0, {"node_rank": 2}), ("high_cpu_g8", 0, {"node_rank": 10})]),
    "mixed_world_candidates": (10_000, [("normal_g8", 0, {}), ("g3", 1, {"local_world_size": 4}),
                                        ("g1", 2, {"local_world_size": 2})]),
}


def identity(k: int, n_nodes: int, overrides=None):
    """Node k's leader in a run of n_nodes x 8 ranks; ``overrides`` replaces fields (node_rank moves
    the global rank with it)."""
    o = dict(overrides or {})
    node = int(o.get("node_rank", k))
    lws = int(o.get("local_world_size", 8))
    ident = {"global_rank": node * 8, "local_rank": 0, "world_size": 8 * n_nodes, "local_world_size": lws,
             "node_rank": node, "hostname": f"h100-node{node}"}
    ident.update({f: v for f, v in o.items() if f not in ("node_rank",)})
    return ident


def make_case(name: str):
    """(window, [raw samples per node], [identity per node])."""
    window, nodes = CASES[name]
    raws = [sc.make_raw(base, seed=seed) for base, seed, _ in nodes]
    idents = [identity(k, len(nodes), o) for k, (_, _, o) in enumerate(nodes)]
    return window, raws, idents


def random_nodes(K: int, seed: int, max_samples: int = 300):
    """K nodes of random size (1 .. max_samples samples, 0 .. 8 GPUs), for the scale tests."""
    import numpy as np

    rng = np.random.default_rng(seed)
    raws, idents = [], []
    for k in range(K):
        G = int(rng.integers(0, 9))
        raws.append(sc.random_raw(int(rng.integers(1, max_samples + 1)), G, seed * 1000 + k))
        idents.append(identity(k, K))
    return raws, idents
