"""Seeded System sample streams (TEST INFRASTRUCTURE): what ``SystemProbe`` would see on a host,
as raw NVML integers (the engine's record) and as the reference's wire rows.  Shared by
``golden/make_system_golden.py`` and the System tests."""
from __future__ import annotations

import numpy as np

MEM_TOTAL = 85_520_809_980   # an 80 GB HBM3 part (divisible by 10: exact threshold cases)
LIMIT_MW = 700_000
RAM_TOTAL = 2_000_000_000_000
IDENTITY = {"global_rank": 0, "local_rank": 0, "world_size": 8, "local_world_size": 8, "node_rank": 0,
            "hostname": "h100-node"}

# name -> (gpus, samples, window, knobs)
CASES = {
    "normal_g8": (8, 240, 10_000, {}),
    "very_high_gpu_memory_g8": (8, 200, 10_000, {"mem_peak": (3, 0.95)}),
    "high_gpu_memory_g8": (8, 200, 10_000, {"mem_peak": (5, 0.85)}),
    "high_gpu_temperature_g8": (8, 200, 10_000, {"temp_peak": (2, 88)}),
    "high_gpu_power_g8": (8, 200, 10_000, {"power_frac": (6, 0.86)}),
    "high_host_memory_g8": (8, 200, 10_000, {"ram_peak": 0.87}),
    "high_cpu_g8": (8, 200, 10_000, {"cpu": 86.0}),
    "low_gpu_utilization_g3": (3, 200, 10_000, {"util": 12}),
    "several_issues_g8": (8, 300, 10_000, {"mem_peak": (1, 0.93), "temp_peak": (4, 91), "power_frac": (7, 0.9),
                                           "ram_peak": 0.9, "cpu": 88.0, "util": 9}),
    "cpu_only": (0, 150, 10_000, {"no_nvml": True}),
    "failed_gpu_g4": (4, 120, 10_000, {"failed": 2}),
    "g1": (1, 100, 10_000, {}),
    "g3": (3, 100, 10_000, {}),
    "g16": (16, 100, 10_000, {}),
    "single_sample_g8": (8, 1, 10_000, {}),
    "window_smaller_g8": (8, 500, 64, {"cpu": 85.0, "late_calm": True}),
    "power_limit_zero_g4": (4, 100, 10_000, {"limit_zero": (1, 3)}),
    "on_threshold_g4": (4, 50, 10_000, {"threshold": True}),
    "no_data": (8, 0, 10_000, {}),
}


def make_raw(name: str, seed: int = 0):
    """List of samples: dict(seq, ts, cpu, ram_used, ram_total, gpu_available, gpu_count,
    gpus=[(util, mem_used, mem_total, temp_c, power_mw, power_limit_mw), ...])."""
    G, n, _, k = CASES[name]
    rng = np.random.default_rng((sum(map(ord, name)) * 7919 + seed) % (1 << 32))
    out = []
    for i in range(n):
        cpu = round(float(rng.uniform(20.0, 60.0)), 1) if "cpu" not in k else float(k["cpu"])
        if k.get("late_calm") and i < n - 64:
            cpu = 10.0  # only the latest W samples are busy: the window must cut
        ram = int(RAM_TOTAL * float(rng.uniform(0.3, 0.6)))
        if "ram_peak" in k and i == n // 2:
            ram = int(RAM_TOTAL * k["ram_peak"])
        gpus = []
        for g in range(G):
            util = int(rng.integers(70, 100)) if "util" not in k else int(k["util"] + rng.integers(0, 3))
            used = int(MEM_TOTAL * float(rng.uniform(0.35, 0.6)))
            temp = int(rng.integers(45, 75))
            limit = LIMIT_MW
            mw = int(rng.integers(150_000, 420_000))
            if "mem_peak" in k and k["mem_peak"][0] == g and i == n // 3:
                used = int(MEM_TOTAL * k["mem_peak"][1])
            if "temp_peak" in k and k["temp_peak"][0] == g and i == n // 4:
                temp = int(k["temp_peak"][1])
            if "power_frac" in k and k["power_frac"][0] == g:
                mw = int(LIMIT_MW * k["power_frac"][1]) + int(rng.integers(-2000, 2000))
            if "limit_zero" in k and g in k["limit_zero"]:
                limit = 0
            if k.get("threshold"):
                util, temp = 30, 85 if g == 0 else 60
                used = MEM_TOTAL // 2 if g else int(MEM_TOTAL * 9 // 10)
                mw = 560_000 if g == 1 else 200_000  # 80 % of the limit, exactly
            if k.get("failed") == g:
                util = used = temp = mw = limit = 0
                gpus.append((0, 0, 0, 0, 0, 0))
                continue
            gpus.append((util, used, MEM_TOTAL, temp, mw, limit))
        if k.get("threshold"):
            cpu, ram = 80.0, RAM_TOTAL // 10 * 8 if i == 0 else RAM_TOTAL // 2
        no_nvml = k.get("no_nvml", False)
        out.append({"seq": i + 1, "ts": 1_760_000_000.0 + 0.5 * i + float(rng.uniform(0, 0.01)), "cpu": cpu,
                    "ram_used": ram, "ram_total": RAM_TOTAL, "gpu_available": not no_nvml,
                    "gpu_count": 0 if no_nvml else G, "gpus": [] if no_nvml else gpus})
    return out


def random_raw(n: int, G: int, seed: int, adversarial: bool = False):
    """n samples of G GPUs with arbitrary (not one-decimal) cpu values; ``adversarial`` mixes
    binades and integer-valued cpu readings."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        cpu = float(rng.uniform(0.0, 100.0))
        if adversarial:
            cpu = float(rng.choice([cpu, cpu * 1e-9, round(cpu), cpu * 1e3 % 100.0, 0.1 * (i % 7)]))
        gpus = [(int(rng.integers(0, 101)), int(rng.integers(0, MEM_TOTAL)), MEM_TOTAL, int(rng.integers(30, 95)),
                 int(rng.integers(50_000, LIMIT_MW)), LIMIT_MW if g % 5 else int(rng.integers(0, LIMIT_MW)))
                for g in range(G)]
        out.append({"seq": i + 1, "ts": 1_760_000_000.0 + 0.5 * i, "cpu": cpu,
                    "ram_used": int(rng.integers(0, RAM_TOTAL)), "ram_total": RAM_TOTAL,
                    "gpu_available": G > 0, "gpu_count": G, "gpus": gpus})
    return out


def wire_row(s):
    """SystemSample.to_wire of one raw sample (what SystemProbe hands the sinks)."""
    return {"seq": s["seq"], "ts": s["ts"], "cpu": s["cpu"], "ram_used": float(s["ram_used"]),
            "ram_total": float(s["ram_total"]), "gpu_available": s["gpu_available"], "gpu_count": s["gpu_count"],
            "gpus": [[float(u), float(m), float(t_), float(c), float(mw / 1000.0), float(lm / 1000.0)]
                     for (u, m, t_, c, mw, lm) in s["gpus"]]}


def sys_records(raw):
    """The engine's records (ctypes array of ``_abi.SysRecord``)."""
    from traceml_b200 import _abi
    from traceml_b200.samplers import sys_record

    arr = (_abi.SysRecord * max(1, len(raw)))()
    for i, s in enumerate(raw):
        arr[i] = sys_record(s["seq"], s["ts"], s["cpu"], s["ram_used"], s["ram_total"], s["gpu_available"],
                            s["gpu_count"], s["gpus"])
    return arr if raw else (_abi.SysRecord * 0)()


def sys_agg_from_oracle(sec):
    """The tml_sys_agg the kernel must produce, from the oracle's section (CPU tests feed the rule
    engine with it)."""
    from traceml_b200 import _abi

    a = _abi.SysAgg()
    ag = sec["aggregate"]
    a.n = ag["system_samples"]
    if not a.n:
        return a
    node = next(iter(sec["nodes"].values()))
    a.first_ts, a.last_ts = ag["first_ts"], ag["last_ts"]
    a.cpu_avg, a.cpu_peak = ag["cpu_avg_percent"], ag["cpu_peak_percent"]
    a.ram_avg, a.ram_peak, a.ram_total = ag["ram_avg_bytes"], ag["ram_peak_bytes"], ag["ram_total_bytes"]
    a.gpu_available, a.gpu_count = int(bool(ag["gpu_available"])), int(ag["gpu_count"])
    if ag["gpu_util_avg_percent"] is not None:
        a.n_gpu = 1  # only "some sample had GPUs" matters to the rule engine
        a.gpu_util_avg, a.gpu_util_peak = ag["gpu_util_avg_percent"], ag["gpu_util_peak_percent"]
        a.gpu_mem_avg, a.gpu_mem_peak = ag["gpu_mem_avg_bytes"], ag["gpu_mem_peak_bytes"]
        a.gpu_temp_avg, a.gpu_temp_peak = ag["gpu_temp_avg_c"], ag["gpu_temp_peak_c"]
        a.gpu_power_avg, a.gpu_power_peak = ag["gpu_power_avg_w"], ag["gpu_power_peak_w"]
    a.n_gpus = len(node["per_gpu"])
    for i, g in node["per_gpu"].items():
        q = a.gpu[int(i)]
        q.n = 1
        q.util_avg, q.util_peak = g["util_avg_percent"], g["util_peak_percent"]
        q.mem_avg, q.mem_peak, q.mem_total = g["mem_avg_bytes"], g["mem_peak_bytes"], g["mem_total_bytes"]
        q.temp_avg, q.temp_peak = g["temp_avg_c"], g["temp_peak_c"]
        q.power_avg, q.power_peak, q.power_limit = g["power_avg_w"], g["power_peak_w"], g["power_limit_w"]
    return a
