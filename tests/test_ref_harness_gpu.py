"""The reference's OWN harness binaries (compiled from /root/reference sources into oracle/_ref/ by
`make -C how-to-optimize-gemm_b200 refharness`), linked against our MY_MMult shims, run on the GPU:
this is the drop-in claim of SURVEY §8b checked end to end.  Skipped where the prebuilt binaries
are absent."""
import os
import re
import subprocess

import pytest

import _libs

pytestmark = pytest.mark.gpu
REFDIR = os.path.join(_libs.ROOT, "oracle", "_ref")


def run(name, *args, env=None, timeout=600):
    exe = os.path.join(REFDIR, name)
    if not os.path.exists(exe):
        pytest.skip(f"{exe} not built")
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout, env=e)


def rows(stdout):
    body = stdout.split("MY_MMult = [")[1].split("];")[0]
    return [ln.split() for ln in body.strip().splitlines() if ln.strip()]


@pytest.mark.parametrize("mode", ["default", "0", "1", "2", "5"])   # shim default (AUTO -> F16X2), STRICT, TF32, BF16X3, F16X2
def test_cuda_harness_unmodified(mode):
    """cuda/test_MMult.cpp + REF_MMult.cpp (OpenBLAS) + compare_matrices.cpp, N = 256..4096 step 256.  "default" is
    what bench.py measures: the shim passes B200_F32_AUTO and no environment override is set."""
    env = {k: v for k, v in os.environ.items() if k != "B200GEMM_F32_MODE"}
    if mode != "default":
        env["B200GEMM_F32_MODE"] = mode
    exe = os.path.join(REFDIR, "ref_cuda_test_MMult__b200.x")
    if not os.path.exists(exe):
        pytest.skip(f"{exe} not built")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert re.search(r'GPU Device 0: ".*" with compute capability 9\.0', r.stdout)
    rs = rows(r.stdout)
    assert [int(x[0]) for x in rs] == list(range(256, 4097, 256))
    for n, gflops, diff in rs:
        assert float(gflops) > 0
        # gate: cuda/test_MMult.cpp:124 (0.5); the fp32-class modes sit at OpenBLAS's own summation-order noise
        assert float(diff) < (0.5 if mode == "1" else 2e-3)


@pytest.mark.parametrize("name", ["MMult_cuBLAS_1", "MMult_cuBLAS_2"])
def test_reference_cublas_comparators_run(name):
    """The reference's own comparators (cuda/MMult_cuBLAS_1.cpp: cublasSgemm; cuda/MMult_cuBLAS_2.cpp:22-25:
    cublasGemmEx CUBLAS_COMPUTE_32F) through the same unmodified harness: the OLD curve of its OLD/NEW plots."""
    r = run(f"ref_cuda_test_MMult__{name}.x")
    assert r.returncode == 0, r.stdout + r.stderr
    rs = rows(r.stdout)
    assert [int(x[0]) for x in rs] == list(range(256, 4097, 256))
    assert all(float(g) > 0 and float(d) < 0.5 for _, g, d in rs)


def test_aarch64_harness_config1():
    """aarch64/test_MMult.cpp at 256^3 through the 9-arg host shim (C += A*B), diff must be 0."""
    r = run("ref_a64_test_MMult__b200.x", env={"B200GEMM_F32_MODE": "0"})
    assert r.returncode == 0, r.stdout + r.stderr
    rs = rows(r.stdout)
    assert len(rs) == 1 and int(rs[0][0]) == 256 and float(rs[0][2]) == 0.0


@pytest.mark.parametrize("mnk", [None, ("64", "64", "64"), ("33", "130", "65"), ("512", "768", "1024")])
def test_int8_harness(mnk):
    """aarch64-int8/test_MMult.c: exits silently (no row printed) on ANY mismatch (test_MMult.c:108-111)."""
    r = run("ref_i8_test_MMult__b200.x", *(mnk or ()))
    assert r.returncode == 0, r.stdout + r.stderr
    rs = rows(r.stdout)
    assert len(rs) == 1 and int(rs[0][2]) == 0
