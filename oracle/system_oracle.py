"""Oracle: System section window + aggregates + diagnosis.  TEST INFRASTRUCTURE ONLY.

Restates, for one node (one system source):
  - the writer's per-sample derived GPU columns, ``src/traceml/aggregator/sqlite_writers/system.py:381-474``
    (average / max over the GPUs present, in index order);
  - the loader's window (latest ``max_rows`` samples of the node, id order) and aggregates,
    ``src/traceml/reporting/sections/system/loader.py:97-167,170-359`` with the helpers of
    ``model.py:189-210`` (``sum(list) / len(list)``: CPython's compensated sum);
  - ``diagnose_system``: ``diagnostics/system/context.py:142-373``, ``rules.py:13-310``,
    ``api.py:47-209``, ``policy.py:22-36``, ``diagnostics/bands.py:21-34``.

Input: ``rows`` = the node's system wire rows in insertion order (``SystemSample.to_wire``:
``seq, ts, cpu, ram_used, ram_total, gpu_available, gpu_count, gpus`` with ``gpus`` a list of
``[util, mem_used, mem_total, temp_c, power_w, power_limit_w]``), ``identity`` = the sampler's
envelope identity (``global_rank, local_rank, world_size, local_world_size, node_rank, hostname``).
Output: the dict ``traceml_b200.sections.build_system`` returns.
"""

from __future__ import annotations

import math
from typing import Any, Dict, List, Optional

SYSTEM_ISSUE_PRIORITY = {  # rules.py:273-281
    "VERY_HIGH_GPU_MEMORY": 0, "HIGH_GPU_TEMPERATURE": 1, "HIGH_GPU_MEMORY": 2, "HIGH_GPU_POWER": 3,
    "HIGH_HOST_MEMORY": 4, "HIGH_CPU": 5, "LOW_GPU_UTILIZATION": 6,
}
SEVERITY_RANK = {"crit": 2, "warn": 1, "info": 0}  # diagnostics/common.py:98-102


def _avg(vals):  # model.py:189-192
    nums = [float(v) for v in vals if v is not None]
    return sum(nums) / len(nums) if nums else None


def _max(vals):  # model.py:195-198
    nums = [float(v) for v in vals if v is not None]
    return max(nums) if nums else None


def _max_int(vals):  # model.py:201-204
    nums = [int(v) for v in vals if v is not None]
    return max(nums) if nums else None


def _min(vals):  # model.py:207-210
    nums = [float(v) for v in vals if v is not None]
    return min(nums) if nums else None


def derived_row(row: Dict[str, Any]) -> Dict[str, Any]:
    """system.py:381-474: the sample's columns as the writer stores them."""
    utils, mems, temps, powers = [], [], [], []
    for g in row.get("gpus") or []:
        if not (isinstance(g, list) and len(g) >= 6):
            continue
        utils.append(float(g[0])); mems.append(float(g[1])); temps.append(float(g[3])); powers.append(float(g[4]))
    return {
        "ts": float(row["ts"]), "cpu": float(row["cpu"]), "ram_used": float(row["ram_used"]),
        "ram_total": float(row["ram_total"]), "gpu_available": bool(row["gpu_available"]),
        "gpu_count": int(row["gpu_count"]),
        "util_avg": sum(utils) / len(utils) if utils else None, "util_peak": max(utils) if utils else None,
        "mem_avg": sum(mems) / len(mems) if mems else None, "mem_peak": max(mems) if mems else None,
        "temp_avg": sum(temps) / len(temps) if temps else None, "temp_peak": max(temps) if temps else None,
        "power_avg": sum(powers) / len(powers) if powers else None, "power_peak": max(powers) if powers else None,
    }


def aggregate(rows: List[Dict[str, Any]]) -> Dict[str, Any]:
    """loader.py:97-125 over the derived rows."""
    d = [derived_row(r) for r in rows]
    return {
        "first_ts": _min(x["ts"] for x in d), "last_ts": _max(x["ts"] for x in d), "system_samples": len(d),
        "cpu_avg_percent": _avg(x["cpu"] for x in d), "cpu_peak_percent": _max(x["cpu"] for x in d),
        "ram_avg_bytes": _avg(x["ram_used"] for x in d), "ram_peak_bytes": _max(x["ram_used"] for x in d),
        "ram_total_bytes": _max(x["ram_total"] for x in d),
        "gpu_available": any(x["gpu_available"] for x in d) if d else None,
        "gpu_count": _max_int(x["gpu_count"] for x in d),
        "gpu_util_avg_percent": _avg(x["util_avg"] for x in d), "gpu_util_peak_percent": _max(x["util_peak"] for x in d),
        "gpu_mem_avg_bytes": _avg(x["mem_avg"] for x in d), "gpu_mem_peak_bytes": _max(x["mem_peak"] for x in d),
        "gpu_temp_avg_c": _avg(x["temp_avg"] for x in d), "gpu_temp_peak_c": _max(x["temp_peak"] for x in d),
        "gpu_power_avg_w": _avg(x["power_avg"] for x in d), "gpu_power_peak_w": _max(x["power_peak"] for x in d),
    }


def per_gpu(rows: List[Dict[str, Any]]) -> Dict[int, Dict[str, Any]]:
    """loader.py:128-156: GPU rows grouped by index (seq, gpu_idx order)."""
    grouped: Dict[int, List[List[float]]] = {}
    for r in rows:
        for i, g in enumerate(r.get("gpus") or []):
            if isinstance(g, list) and len(g) >= 6:
                grouped.setdefault(i, []).append([float(v) for v in g[:6]])
    out = {}
    for i, gs in sorted(grouped.items()):
        out[i] = {"gpu_idx": i,
                  "util_avg_percent": _avg(g[0] for g in gs), "util_peak_percent": _max(g[0] for g in gs),
                  "mem_avg_bytes": _avg(g[1] for g in gs), "mem_peak_bytes": _max(g[1] for g in gs),
                  "mem_total_bytes": _max(g[2] for g in gs),
                  "temp_avg_c": _avg(g[3] for g in gs), "temp_peak_c": _max(g[3] for g in gs),
                  "power_avg_w": _avg(g[4] for g in gs), "power_peak_w": _max(g[4] for g in gs),
                  "power_limit_w": _max(g[5] for g in gs)}
    return out


# ----------------------------------------------------------------------------- diagnosis
def _classify(v, low_below=None, high_at=None, very_high_at=None) -> Optional[str]:  # bands.py:21-34
    if v is None:
        return None
    v = float(v)
    if very_high_at is not None and v >= very_high_at:
        return "very_high"
    if high_at is not None and v >= high_at:
        return "high"
    if low_below is not None and v < low_below:
        return "low"
    return "normal"


def _fraction(num, den):  # context.py:154-164
    if num is None or den is None or float(den) <= 0.0:
        return None
    return max(0.0, float(num) / float(den))


def _best_idx(gpus, key, highest):  # context.py:175-202
    best_idx, best = None, None
    for i, g in gpus.items():
        v = g.get(key)
        if v is None:
            continue
        if best is None or (highest and v > best) or (not highest and v < best):
            best_idx, best = int(i), v
    return best_idx


def _best_pressure_idx(gpus, num_key, den_key):  # context.py:263-282
    best_idx, best = None, None
    for i, g in gpus.items():
        v = _fraction(g.get(num_key), g.get(den_key))
        if v is None:
            continue
        if best is None or v > best:
            best_idx, best = int(i), v
    return best_idx


def _pct(v):  # rules.py:13-14
    return "n/a" if v is None else f"{float(v):.1f}%"


def _sfx(i):  # rules.py:17-18
    return "" if i is None else f" on gpu{int(i)}"


def _node_rules(agg: Dict[str, Any], gpus: Dict[int, Dict[str, Any]]) -> List[Dict[str, Any]]:
    """context.py:285-373 + rules.py:55-259 for one node."""
    mem_fracs = [f for f in (_fraction(g["mem_peak_bytes"], g["mem_total_bytes"]) for g in gpus.values()) if f is not None]
    pow_fracs = [f for f in (_fraction(g["power_avg_w"], g["power_limit_w"]) for g in gpus.values()) if f is not None]
    ram_frac = _fraction(agg["ram_peak_bytes"], agg["ram_total_bytes"])
    mem_pct = max(mem_fracs) * 100.0 if mem_fracs else None
    pow_pct = max(pow_fracs) * 100.0 if pow_fracs else None
    ram_pct = ram_frac * 100.0 if ram_frac is not None else None
    mem_idx = _best_pressure_idx(gpus, "mem_peak_bytes", "mem_total_bytes")
    pow_idx = _best_pressure_idx(gpus, "power_avg_w", "power_limit_w")
    temp_idx = _best_idx(gpus, "temp_peak_c", True)
    util_idx = _best_idx(gpus, "util_avg_percent", False)
    temp, cpu, util = agg["gpu_temp_peak_c"], agg["cpu_avg_percent"], agg["gpu_util_avg_percent"]

    def issue(kind, status, sev, summary, action, metric, phase, score, gpu, evidence):
        return {"kind": kind, "status": status, "severity": sev, "summary": summary, "action": action,
                "metric": metric, "phase": phase, "score": float(score) if score is not None else None,
                "share_pct": None, "skew_pct": None, "ranks": [] if gpu is None else [int(gpu)],
                "evidence": evidence}

    out = []
    band = _classify(mem_pct, 30.0, 80.0, 90.0)
    if band == "very_high":
        out.append(issue("VERY_HIGH_GPU_MEMORY", "VERY HIGH GPU MEMORY", "crit",
                         f"GPU memory was very high, peaking at {_pct(mem_pct)}{_sfx(mem_idx)}.",
                         "Reduce GPU memory pressure before scaling this run.", "gpu_mem_peak_percent", "gpu_memory",
                         mem_pct, mem_idx, {"gpu_mem_peak_percent": mem_pct, "gpu_idx": mem_idx}))
    if _classify(temp, high_at=85.0) == "high":
        out.append(issue("HIGH_GPU_TEMPERATURE", "HIGH GPU TEMPERATURE", "crit",
                         f"GPU temperature was high, peaking at {float(temp):.1f} C{_sfx(temp_idx)}.",
                         "Check cooling and thermal throttling risk.", "gpu_temp_peak_c", "gpu_temperature",
                         float(temp), temp_idx, {"gpu_temp_peak_c": float(temp), "gpu_idx": temp_idx}))
    if band == "high":
        out.append(issue("HIGH_GPU_MEMORY", "HIGH GPU MEMORY", "warn",
                         f"GPU memory was high, peaking at {_pct(mem_pct)}{_sfx(mem_idx)}.",
                         "Watch GPU memory headroom for larger batches or models.", "gpu_mem_peak_percent",
                         "gpu_memory", mem_pct, mem_idx, {"gpu_mem_peak_percent": mem_pct, "gpu_idx": mem_idx}))
    if _classify(pow_pct, 30.0, 80.0) == "high":
        out.append(issue("HIGH_GPU_POWER", "HIGH GPU POWER", "warn",
                         f"GPU power was high, averaging {_pct(pow_pct)} of limit{_sfx(pow_idx)}.",
                         "Review power headroom if this run is unstable.", "gpu_power_avg_limit_percent", "gpu_power",
                         pow_pct, pow_idx, {"gpu_power_avg_limit_percent": pow_pct, "gpu_idx": pow_idx}))
    if _classify(ram_pct, 30.0, 80.0) == "high":
        out.append(issue("HIGH_HOST_MEMORY", "HIGH HOST MEMORY", "warn",
                         f"Host RAM usage was high, peaking at {_pct(ram_pct)} of total.",
                         "Reduce host memory pressure or inspect data workers.", "ram_peak_percent", "ram", ram_pct,
                         None, {"ram_peak_percent": ram_pct}))
    if _classify(cpu, 30.0, 80.0) == "high":
        out.append(issue("HIGH_CPU", "HIGH CPU", "warn", f"CPU usage was high, averaging {_pct(cpu)}.",
                         "Inspect CPU-side preprocessing or host contention.", "cpu_avg_percent", "cpu", cpu, None,
                         {"cpu_avg_percent": cpu}))
    if _classify(util, 30.0, 80.0) == "low":
        out.append(issue("LOW_GPU_UTILIZATION", "LOW GPU UTILIZATION", "info",
                         f"GPU utilization was low, averaging {_pct(util)}.",
                         "Use step-time diagnostics to check host or input stalls.", "gpu_util_avg_percent",
                         "gpu_utilization", 100.0 - float(util), util_idx,
                         {"gpu_util_avg_percent": util, "lowest_util_gpu_idx": util_idx}))
    return sorted(out, key=lambda i: (SYSTEM_ISSUE_PRIORITY.get(i["kind"], 999), -(i["score"] or 0.0)))


def _scope(label, node_rank, issue):  # api.py:106-134
    scope = {"level": "node", "node": label, "node_rank": node_rank}
    text = issue["summary"]
    if issue["ranks"]:
        g = int(issue["ranks"][0])
        scope["level"], scope["gpu_idx"] = "gpu", g
        existing, suffix = f" on gpu{g}", f" on {label} gpu{g}"
        text = text.replace(existing, suffix) if existing in text else f"{text.rstrip('.')}{suffix}."
    elif label:
        text = f"{text.rstrip('.')} on {label}."
    return scope, text


def diagnose(agg, nodes) -> Dict[str, Any]:
    """api.py:189-209."""
    issues = []
    for node in nodes.values():
        if node["aggregate"]["system_samples"] <= 0:
            continue
        ident = node["identity"]
        for i in _node_rules(node["aggregate"], node["per_gpu"]):
            scope, text = _scope(ident["label"], ident["node_rank"], i)
            i = dict(i, summary=text, evidence=dict(i["evidence"], scope=scope,
                                                     samples_used=int(node["aggregate"]["system_samples"])))
            issues.append(i)
    issues.sort(key=lambda i: (SYSTEM_ISSUE_PRIORITY.get(i["kind"], 999), -SEVERITY_RANK.get(i["severity"], 0),
                               -float(i["score"] or 0.0), str(i["evidence"]["scope"].get("node") or "")))
    if issues:
        t = issues[0]
        primary = {"severity": t["severity"], "status": t["status"], "reason": t["summary"], "action": t["action"],
                   "kind": t["kind"], "samples_used": int(t["evidence"].get("samples_used") or 0),
                   "scope": dict(t["evidence"]["scope"])}
    elif agg["system_samples"] <= 0:
        primary = {"severity": "info", "status": "NO DATA", "reason": "No system telemetry was recorded.",
                   "action": "Collect system telemetry for host-level context.", "kind": "NO_DATA",
                   "samples_used": agg["system_samples"], "scope": {"level": "cluster"}}
    else:  # cluster signals have no per-GPU rows (context.py:291-293)
        gpu = agg["gpu_util_avg_percent"] is not None or agg["gpu_temp_peak_c"] is not None
        primary = {"severity": "info", "status": "NORMAL",
                   "reason": "CPU, RAM, and GPU showed no system pressure." if gpu
                   else "CPU and RAM showed no system pressure.",
                   "action": "Use training diagnostics for model-level bottlenecks.", "kind": "NORMAL",
                   "samples_used": agg["system_samples"], "scope": {"level": "cluster"}}
    return {"primary": primary, "issues": issues}


def system_section(rows: List[Dict[str, Any]], identity: Dict[str, Any], max_rows: int) -> Dict[str, Any]:
    """The whole section for one node: the latest ``max_rows`` samples (loader.py:170-193)."""
    win = list(rows)[-int(max_rows):] if max_rows > 0 else []
    agg = aggregate(win)
    nodes = {}
    expected = 1
    if win:
        label = str(int(identity["node_rank"])) if identity.get("node_rank") is not None \
            else str(int(identity.get("global_rank") or 0))
        ident = {"label": label}
        ident.update({k: identity.get(k) for k in ("node_rank", "hostname", "global_rank", "local_rank",
                                                   "local_world_size", "world_size")})
        nodes[label] = {"identity": ident, "aggregate": aggregate(win), "per_gpu": per_gpu(win)}
        if identity.get("world_size") and identity.get("local_world_size"):  # loader.py:159-167
            expected = max(1, int(math.ceil(float(identity["world_size"]) / float(identity["local_world_size"]))))
    return {"aggregate": agg, "nodes": nodes, "expected_nodes": expected, "diagnosis": diagnose(agg, nodes)}
