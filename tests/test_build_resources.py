"""Resource budget of the compiled kernels, from the `-Xptxas -v` log the in-tree build writes
(how-to-optimize-gemm_b200/build_ptxas.log): the occupancy each kernel is designed for (DESIGN §4) only holds
while these stay true.  CPU only (ptxas cross-compiles sm_90a without a GPU)."""
import os
import re

import _libs

LOG = os.path.join(_libs.ROOT, _libs.PKG, "build_ptxas.log")


def kernels():
    if not os.path.exists(LOG):      # the log is a build product (git-ignored): regenerate it with the library
        import subprocess
        subprocess.check_call(["make", "-B", "-C", os.path.join(_libs.ROOT, _libs.PKG), "libb200gemm.so"])
    out, name = {}, None
    for line in open(LOG):
        m = re.search(r"Compiling entry function '(\w+)' for 'sm_90a'", line)
        if m:
            name = m.group(1)
            out[name] = {"regs": None, "spill": None}
        elif name and "spill stores" in line:
            out[name]["spill"] = int(re.search(r"(\d+) bytes spill stores", line).group(1))
        elif name and "Used" in line and "registers" in line:
            out[name]["regs"] = int(re.search(r"Used (\d+) registers", line).group(1))
    return out


def test_log_covers_every_kernel_family():
    k = kernels()
    for frag in ["gemm_tc_kernel", "gemm_ffma_kernel", "gemm_ffma_fat_kernel", "gemm_generic_kernel", "split_planes_kernel"]:
        assert any(frag in n for n in k), frag
    assert all(v["regs"] is not None and v["spill"] is not None for v in k.values())


def test_tensor_core_kernels_do_not_spill():
    # one CTA of 384 threads per SM (168 registers at launch; setmaxnreg 40 for the producer warpgroup, 232 for
    # the two consumers): the running sum of a split-precision tile lives in the consumers' registers — a spill
    # there would sit in the per-chunk add loop
    for n, v in kernels().items():
        if "gemm_tc_kernel" in n:
            # <= 48 bytes: a few split kernels keep the mbarrier watchdog's clock value in one stack slot
            # (LDL/STL only on the slow path of a wait); nothing from the accumulation loops may spill
            assert v["spill"] <= 48 and v["regs"] <= 255, (n, v)
            if "ProdX" in n:
                assert v["regs"] <= 168, (n, v)


def test_strict_kernels_keep_their_occupancy():
    k = kernels()
    thin = next(v for n, v in k.items() if "gemm_ffma_kernel" in n)
    fat = next(v for n, v in k.items() if "gemm_ffma_fat_kernel" in n)
    assert thin["regs"] <= 128           # 256 threads x 2 CTAs/SM x 128 = the whole register file
    assert thin["spill"] <= 64           # the C += entry's prologue only; the k loop must stay in registers
    assert fat["regs"] <= 255 and fat["spill"] == 0


def test_prepass_kernels_allow_full_occupancy():
    for n, v in kernels().items():
        if "split_planes_kernel" in n or "split_f16_cols_kernel" in n or "col_absmax_kernel" in n:
            assert v["regs"] <= 64 and v["spill"] == 0, (n, v)      # 8 blocks of 256 threads per SM
        if "split_f16_rows_kernel" in n:
            assert v["spill"] == 0, (n, v)                          # register-resident rows: no local memory
