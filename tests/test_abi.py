"""The drop-in boundary without a GPU: the C-ABI library loads, exports exactly what
include/b200gemm.h declares, and refuses to compute (loudly) when there is no sm_90 device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import _libs

HDR = os.path.join(_libs.ROOT, "include", "b200gemm.h")


def declared_functions():
    src = open(HDR).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_\w+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    fns = declared_functions()
    for must in ["b200_gemm_f32", "b200_gemm_f32_host", "b200_gemm_bf16", "b200_gemm_s8s32",
                 "b200_gemm_s8s32_host", "b200_convert_f32_to_bf16"]:
        assert must in fns


def test_library_exports_every_declared_symbol(gemm):
    for fn in declared_functions():
        assert hasattr(gemm.lib, fn), f"{fn} declared in include/b200gemm.h but not exported"
    assert sorted(gemm.EXPORTS) == declared_functions()


def test_library_exports_nothing_undeclared(gemm):
    """Every b200_* symbol the shared object exports is declared (and documented) in the header."""
    out = subprocess.check_output(["nm", "-D", "--defined-only", gemm.LIB_PATH], text=True)
    exported = sorted({ln.split()[-1] for ln in out.splitlines() if " T b200_" in ln})
    assert exported == declared_functions()


def test_no_undefined_oracle_or_blas_dependencies(gemm):
    """The product must not link the oracle, the reference, cuBLAS or any BLAS."""
    out = subprocess.check_output(["ldd", gemm.LIB_PATH], text=True)
    for bad in ["oracle", "libref", "cublas", "openblas", "cutlass"]:
        assert bad not in out.lower(), out
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", gemm.LIB_PATH], text=True)
    assert "oracle_" not in syms and "cblas_" not in syms and "cublas" not in syms.lower()


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_fails_loudly_without_device(gemm):
    assert gemm.lib.b200_gemm_device_ok() == -2
    a = np.ones((4, 4), np.float32)
    with pytest.raises(gemm.B200GemmError) as e:
        gemm.MY_MMult(4, 4, 4, a, 4, a, 4, a.copy(), 4)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)
    i8 = np.ones((4, 4), np.int8)
    with pytest.raises(gemm.B200GemmError):
        gemm.MY_MMult_int8(4, 4, 4, i8, 4, i8, 4, np.zeros((4, 4), np.int32), 4)


def test_argument_validation(gemm):
    lib = gemm.lib
    assert lib.b200_gemm_f32(-1, 4, 4, None, 4, None, 4, None, 4, 0, None) == -1
    assert lib.b200_gemm_f32(4, 4, 4, None, 4, None, 4, None, 4, 0, None) == -1      # null C
    buf = (C.c_float * 64)()
    assert lib.b200_gemm_f32(4, 4, 4, buf, 2, buf, 4, buf, 4, 0, None) == -1          # lda < k
    assert lib.b200_gemm_f32(4, 4, 4, buf, 4, buf, 4, buf, 3, 0, None) == -1          # ldc < n
    assert lib.b200_gemm_f32(0, 4, 4, None, 4, None, 4, None, 4, 0, None) == 0        # empty: no-op
    assert lib.b200_gemm_s8s32(4, 0, 4, None, 4, None, 4, None, 4, None) == 0
    assert lib.b200_gemm_bf16(4, 4, 4, buf, 4, buf, 4, buf, 4, 7, None) == -1         # bad out_type
    assert lib.b200_gemm_s8s8_requant(4, 4, 4, buf, 4, buf, 4, buf, 4, None, None, None) == -1   # scales are required
    assert lib.b200_gemm_s8s8_requant(4, 4, 4, buf, 4, buf, 4, buf, 3, buf, None, None) == -1    # ldc < n
    assert lib.b200_gemm_s8s8_requant(0, 4, 4, None, 4, None, 4, None, 4, None, None, None) == 0  # empty: no-op
    h = C.c_void_p()
    assert lib.b200_gemm_f32_pack_b(4, 4, None, 4, 2, C.byref(h), None) == -1 and not h.value   # null B
    assert lib.b200_gemm_f32_pack_b(4, 4, buf, 4, 0, C.byref(h), None) == -3                     # STRICT has no split
    assert lib.b200_gemm_f32_packed(4, 4, 4, buf, 4, None, buf, 4, 0, None) == -1                # null handle
    lib.b200_gemm_f32_pack_free(None)                                                            # no-op
    assert b"bad argument" in lib.b200_gemm_strerror(-1)


def test_shim_objects_define_the_reference_symbols():
    """shim/*.o must define the exact (mangled) MY_MMult symbols the reference harnesses reference
    (SURVEY §8b): 10-arg cuda form, 9-arg CPU form, C-linkage int8 form."""
    d = os.path.join(_libs.ROOT, _libs.PKG, "shim")
    if not os.path.exists(os.path.join(d, "MY_MMult_b200.o")):
        subprocess.check_call(["make", "-C", os.path.join(_libs.ROOT, _libs.PKG), "host"])
    syms = subprocess.check_output(["nm", os.path.join(d, "MY_MMult_b200.o")], text=True)
    assert " T _Z8MY_MMultP13cublasContextiiiPfiS1_iS1_i" in syms      # cuda/test_MMult.cpp:13
    assert " T _Z8MY_MMultiiiPfiS_iS_i" in syms                        # aarch64/MMult0.cpp:3
    syms8 = subprocess.check_output(["nm", os.path.join(d, "MY_MMult_int8_b200.o")], text=True)
    assert " T MY_MMult" in syms8                                       # aarch64-int8/test_MMult.c:9
