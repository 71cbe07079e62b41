"""CPU test of the bench.py contract: the reference arm runs without a GPU and prints ONE JSON line with the keys the
driver reads; the product arm's JSON line committed under profiles/ carries the same metric/unit/config plus the
`roofline`, `cpu_baseline`, `e2e`, `clocks`, `gpu_launches` objects."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--size", "384", "--steps",
                          "2", "--warmup", "1"], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, GPX_REF_BUDGET_S="60"))
    assert out.returncode == 0, out.stderr
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, out.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "evals/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["dtype"] == "f64" and d["data"] == "synthetic"
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and "sample" in d["cpu_baseline"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert abs(d["e2e"]["value"] - d["value"]) < 1e-12 and d["steps"] >= 1
    assert "workload" in d["config"] and "model" not in d["config"]


def test_non_zero_ranks_of_the_reference_arm_exit_quietly():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--size", "256"],
                         capture_output=True, text=True, timeout=120, env=dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1"))
    assert out.returncode == 0 and out.stdout.strip() == ""


import pytest


@pytest.mark.parametrize("name", ["h100_bench_ours_n16384.json"])
def test_committed_product_line_has_the_contract_keys(name):
    p = os.path.join(ROOT, "profiles", name)
    d = json.loads([l for l in open(p).read().splitlines() if l.startswith("{")][-1])
    assert d["roofline"]["unit"] in ("TFLOP/s", "GB/s") and "peak" in d["roofline"] and "achieved" in d["roofline"]
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and "workload" in d["config"] and "l2" in d["config"]
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "clocks"):
        assert key in d, key
    assert d["roofline"]["bound"] == "tensor" and 0 < d["roofline"]["frac"] < 1.05
    assert d["gpu_launches"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0
    assert d["cpu_baseline"]["parity_vs_gpu"]["lml_abs"] <= 1e-8
    assert d["cpu_baseline"]["parity_vs_gpu"]["grad_rel_max"] <= 1e-6
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
