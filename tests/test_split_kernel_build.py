"""The F16X2 kernel (gemm_tc_split_kernel) keeps its running sum, its chunk accumulator and the k-blocks issued ahead of
a tile's store in registers, and ptxas keeps its wgmma chain asynchronous: a spill would sit in the per-chunk fold,
and a serialised wgmma would run the tensor cores one instruction at a time.  Read from the `-Xptxas -v` log of the
in-tree build; CPU only."""
import re

import test_build_resources as resources


def test_split_kernels_do_not_spill():
    split = {n: v for n, v in resources.kernels().items() if "gemm_tc_split_kernel" in n}
    assert len(split) == 4, sorted(split)                # F16X2 in the four operand layouts
    for n, v in split.items():
        assert v["spill"] == 0 and v["regs"] <= 168, (n, v)


def test_split_kernels_keep_wgmma_asynchronous():
    log = open(resources.LOG).read()
    assert not re.search(r"serialized.*gemm_tc_split_kernel", log)
