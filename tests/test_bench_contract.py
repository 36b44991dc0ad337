"""The bench.py JSON contract, checked on lines bench.py printed on an H100 (tests/golden/bench_line.json: `bench.py --gpus 1 --steps 20
--warmup 3`; bench_reference_line.json: `bench.py --impl reference`) and on the argument parser: a missing key would make a recorded
result unusable."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e"]


def _load(name):
    return json.load(open(os.path.join(ROOT, "tests", "golden", name)))


def test_our_line_has_every_contract_key():
    d = _load("bench_line.json")
    for k in BASE_KEYS + ["clocks", "gpu_launches", "roofline", "cpu_baseline"]:
        assert k in d, k
    assert d["n_gpus"] == 1 and d["higher_is_better"] is True and d["data"] == "synthetic" and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    assert d["warmup"] >= 3 and d["gpu_launches"] == d["roofline"]["launches_per_step"] * d["steps"] > 0
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"], k
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] < d["value"]
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(d["value"] * d["ms_per_step"] - 1000.0) < 1e-6 * 1000                    # tok/s x ms/token
    assert abs(r["achieved"] - r["algorithmic_bytes_per_step"] * d["value"] / 1e9) < 1e-6 * r["achieved"]
    for k in ("sm_mhz", "sm_max_mhz", "reasons"):
        assert k in d["clocks"], k
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    c = d["cpu_baseline"]
    for k in ("value", "unit", "cores", "kind", "sample"):
        assert k in c, k
    assert c["kind"] in ("reference", "port")
    pp = d["pp512"]
    assert pp["roofline"]["bound"] == "tensor" and pp["e2e"]["h2d_bytes_per_step"] == 512 * 4096 * 4


def test_reference_line_contract():
    d = _load("bench_reference_line.json")
    for k in BASE_KEYS + ["impl", "cpu_baseline"]:
        assert k in d, k
    assert d["impl"] == "reference" and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["e2e"]["value"] == d["value"] == d["cpu_baseline"]["value"]
    ours = _load("bench_line.json")
    assert d["metric"] == ours["metric"] and d["unit"] == ours["unit"] and d["config"]["workload"] == ours["config"]["workload"]


def test_bench_cli_defaults():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0
    for flag in ("--gpus", "--steps", "--warmup", "--impl", "--dump-outputs"):
        assert flag in out.stdout, flag
