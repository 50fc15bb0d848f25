"""bench.py's driver contract, CPU side: the reference arm runs without a GPU and prints exactly one
JSON line with the keys the driver reads; the GPU arm's source carries every required key."""
import json
import os
import subprocess
import sys
import pytest

import _libs


def test_reference_arm_prints_one_json_line():
    env = dict(os.environ, OPENBLAS_NUM_THREADS="8")
    r = subprocess.run([sys.executable, os.path.join(_libs.ROOT, "bench.py"), "--impl", "reference", "--gpus", "1",
                        "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "GFLOP/s" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["value"] > 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "4096" in d["config"]["workload"]


def test_reference_arm_survives_the_torchrun_environment():
    """Round-1 SCALE run: under torchrun (OMP_NUM_THREADS=1 exported into every rank) the reference arm hung for
    828 s at N=2/4 and crashed at N=8 — growing OpenBLAS-0.2.20's thread pool after load dead-locks.  The arm now
    runs the CPU path in a fresh process whose pool is sized by OPENBLAS_NUM_THREADS at load; same workload string
    as our arm (the driver's same_config check)."""
    if not _libs.have_ref():
        pytest.skip("oracle/_ref/libref.so (the reference's OpenBLAS) not built")
    env = dict(os.environ, OMP_NUM_THREADS="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0", B200_REF_THREADS="128")
    r = subprocess.run([sys.executable, os.path.join(_libs.ROOT, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip())
    assert d["impl"] == "reference" and d["value"] > 0 and d["cpu_baseline"]["cores"] == 128
    sys.path.insert(0, _libs.ROOT)
    import bench
    assert d["config"]["workload"] == bench.workload_str(8192, 4096)


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(_libs.ROOT, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_gpu_arm_emits_contract_keys():
    src = open(os.path.join(_libs.ROOT, "bench.py")).read()
    for key in ['"metric"', '"value"', '"unit"', '"n_gpus"', '"steps"', '"warmup"', '"ms_per_step"', '"higher_is_better"',
                '"scaling"', '"vs_baseline"', '"dtype"', '"data"', '"config"', '"workload"', '"roofline"', '"bound"',
                '"achieved"', '"peak"', '"frac"', '"traffic"', '"cpu_baseline"', '"e2e"', '"h2d_bytes_per_step"',
                '"d2h_bytes_per_step"', '"gpu_launches"', '"clocks"', '"sm_mhz"', '"sm_max_mhz"', '"reasons"', '"verified"',
                '"max_rel_err"', '"c5"', '"configs34"', '"sustained"', '"openblas_1_thread"']:
        assert key in src, key
