"""CPU: bench.py's contract -- the reference arm runs on host cores and prints one JSON line with the agreed
keys; the committed H100 bench line carries every key a consumer of the line reads."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "cpu_baseline"]


def test_reference_arm_prints_contract_line():
    env = dict(os.environ, GPB200_CPU_SAMPLE_N="768")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    for k in REQUIRED:
        assert k in j, k
    assert j["impl"] == "reference" and j["unit"] == "GFLOP/s" and j["higher_is_better"] is True
    assert j["cpu_baseline"]["kind"] == "port" and j["cpu_baseline"]["cores"] >= 1
    assert j["e2e"]["h2d_bytes_per_step"] == 0 and j["gpu_launches"] == 0
    assert j["value"] > 0 and "workload" in j["config"]
    # same config string as our arm; the value is the phase-extrapolated full-config rate, the raw sample rate sits beside it
    assert "N=32768" in j["config"]["workload"] and j["config"]["value_kind"] == "extrapolated_to_full_config"
    assert j["config"]["rate_at_sample_gflops"] > 0 and "N_sample=768" in j["cpu_baseline"]["sample"]


def test_reference_arm_ignores_torchrun_thread_pinning():
    """torchrun exports OMP_NUM_THREADS=1; the CPU arm must still use every host core and say how many."""
    env = dict(os.environ, GPB200_CPU_SAMPLE_N="512", OMP_NUM_THREADS="1", RANK="0", LOCAL_RANK="0", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    j = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][0])
    assert j["cpu_baseline"]["cores"] == (os.cpu_count() or 1)


def test_phase_extrapolation_model():
    import bench
    sec = {"cov_loop": 1.0, "dmll_loop": 2.0, "solve_mll": 0.5, "dpotrf": 3.0, "potrs_identity_ger": 10.0}
    assert abs(bench.extrapolate_full(sec, 8192, 32768) - (3.5 * 16 + 13.0 * 64)) < 1e-9
    assert abs(bench.extrapolate_full(sec, 32768, 32768) - 16.5) < 1e-9


def test_reference_arm_other_ranks_stay_silent():
    env = dict(os.environ, GPB200_CPU_SAMPLE_N="256", RANK="1", LOCAL_RANK="1", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=120, env=env, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.parametrize("name", ["h100_bench_1gpu.json"])
def test_committed_bench_lines_have_every_key(name):
    j = json.load(open(os.path.join(ROOT, "profiles", name)))
    for k in REQUIRED + ["clocks", "roofline"]:
        assert k in j, (name, k)
    assert j["dtype"] == "f64" and j["scaling"] == "strong" and j["data"] == "synthetic"
    assert j["gpu_launches"] > 0 and j["e2e"]["h2d_bytes_per_step"] > 0
    assert not set(j["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    if j["n_gpus"] == 1:
        rf = j["roofline"]
        assert rf["bound"] == "tensor" and rf["unit"] == "TFLOP/s" and 0.5 < rf["frac"] <= 1.05
        assert abs(rf["frac"] - rf["achieved"] / rf["peak"]) < 1e-9
        assert j["cpu_baseline"]["kind"] == "port"
        # value == F_alg / time
        assert abs(j["value"] - (32768.0 ** 3 + 2 * 32768.0 ** 2) / (j["ms_per_step"] * 1e-3) * 1e-9) < 1e-6 * j["value"]
