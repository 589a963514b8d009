"""CPU: the committed bench lines (profiles/h100_bench_*.json, written by bench.py on one H100; see profiles/README.md)
carry every key of the measurement contract, and bench.py's argument surface is the documented one."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILES = os.path.join(ROOT, "profiles")

BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks"}


def load(name):
    path = os.path.join(PROFILES, name)
    if not os.path.exists(path):
        pytest.skip("%s not committed" % name)
    return json.loads(open(path).read().strip().splitlines()[-1])


WORKLOADS = ["c2", "c2g", "c3", "c3d", "c4", "c4d", "c5mb", "c2b", "c5mbb", "c2l", "c5mbl"]
LINES = ["h100_bench_%s.json" % wl for wl in WORKLOADS]


@pytest.mark.parametrize("name", LINES)
def test_bench_line_has_contract_keys(name):
    d = load(name)
    missing = BASE_KEYS - set(d)
    if name != "h100_bench_c2.json":
        missing -= {"cpu_baseline"}          # the other workloads were run with --no-cpu-baseline
    assert not missing, missing
    assert d["higher_is_better"] is True and d["scaling"] == "weak" and d["dtype"] in ("f32", "bf16 i/o, f32 accumulate")
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["gpu_launches"] >= d["steps"]
    assert "workload" in d["config"]
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert 0 < r["frac"] < 1
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and 0 < e["value"] < d["value"]
    c = d["clocks"]
    assert not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert "timed_call" in d and d["roofline"]["kernel_ms"] > 0
    if "cpu_baseline" in d:
        b = d["cpu_baseline"]
        assert b["kind"] in ("port", "reference") and b["cores"] >= 1 and b["value"] > 0 and b["sample"]


def test_round2_both_arms_share_the_config_dict():
    ours, ref = load("h100_bench_c2.json"), load("h100_bench_ref_c2.json")
    assert ref["impl"] == "reference" and ours["config"] == ref["config"] and ours["metric"] == ref["metric"]
    assert set(ref["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"}


def test_reference_arm_line():
    d = load("h100_bench_ref_c2.json")
    assert d["impl"] == "reference" and d["unit"] == "lattices/s"
    ours = load("h100_bench_c2.json")
    assert d["config"]["workload"] == ours["config"]["workload"] and d["metric"] == ours["metric"]
    assert set(d["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"}


def test_bench_cli_surface():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"], capture_output=True, text=True)
    assert out.returncode == 0
    for flag in ("--gpus", "--steps", "--warmup", "--impl"):
        assert flag in out.stdout
