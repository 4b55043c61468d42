"""The JSON lines bench.py printed on one H100 (committed under profiles/) carry every key
of the result line; keeps the line format from drifting.  (bench.py itself needs a GPU;
its output is what can be checked here.)"""

import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step",
             "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e",
             "clocks", "gpu_launches"}


def _line(name):
    text = open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()[-1]
    return json.loads(text)


OURS = "h100_bench_n1.json"


def test_h100_bench_line():
    d = _line(OURS)
    assert BASE_KEYS <= set(d), BASE_KEYS - set(d)
    assert d["n_gpus"] == 1 and d["unit"] == "GB/s" and d["higher_is_better"] is True
    assert d["scaling"] == "weak" and d["vs_baseline"] is None and d["dtype"] == "u8"
    assert d["data"] == "synthetic" and "workload" in d["config"] and "l2" in d["config"]
    assert d["warmup"] >= 3 and d["gpu_launches"] > 0
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    assert d["e2e"]["d2h_bytes_per_step"] == 16_060_522_496
    assert 0 < d["e2e"]["value"] <= d["value"] * 1.02      # e2e cannot beat the raw path
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(r)
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert r["frac"] >= 0.70                                  # north_star: >= 70 % of the HBM roofline
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"])
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown",
                                               "sw_thermal_slowdown"}
    c = d["cpu_baseline"]
    assert {"value", "unit", "cores", "kind", "sample"} <= set(c) and c["kind"] in ("reference", "port")
    assert d["value"] > c["value"]                            # faster than the reference's loop
    assert d["stall_ms"]["async"] < 50.0                      # north_star: < 50 ms stall
    assert d["stall_ms"]["async"] < d["stall_ms"]["blocking"]
    assert {"sm_mhz", "reasons"} <= set(d["stall_ms"]["clocks"])  # clocks of the stall windows
    fresh = d["restore_fresh_process"]
    assert fresh["ours"]["bit_exact_probe"] and fresh["reference_style"]["bit_exact_probe"]
    assert fresh["ours"]["restore_call_s"] < fresh["reference_style"]["restore_call_s"]
    # PCIe Gen5 x16 cannot carry more than ~58 GB/s
    assert d["value"] < 58.0


def test_reference_arm_line():
    d = _line("h100_bench_reference_n1.json")
    assert d["impl"] == "reference" and d["unit"] == "GB/s" and d["metric"] == _line(OURS)["metric"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    assert d["e2e"]["value"] == d["value"]
    assert {"kind", "cores", "sample", "value"} <= set(d["cpu_baseline"])
