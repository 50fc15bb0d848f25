"""Grouped and batched blockwise-scaled FP8 GEMMs (b200_gemm_fp8_blockwise_grouped / _batched) and scaled_grouped_mm()
with blockwise scales: DeepSeek-V3-style FP8 mixture-of-experts layers, activations scaled per 1 x 128 and each expert's
weight per 128 x 128 (or 1 x 128) block, every expert in one launch.

Every group (rows [end_{g-1}, end_g) of A and C, times B_g) and every batch entry is one (N, T) b200_gemm_fp8_blockwise
call with no bias on its own rows, B and scales, so each must equal that call on contiguous copies bit for bit.  Output
buffers start as NaN, the operands' padding holds FP8 NaN bytes and the scale tensors are NaN between their rows and
k-blocks, and whole buffers are compared: a row written to the wrong place, a row past the last group written, or a
padding byte or scale read out of place cannot pass.  On integer operands every block product is exact, and the results
must equal test_fp8_blockwise_gpu's FMA-chain oracle bit for bit.

The argument checks, scaled_grouped_mm's recipe resolution and refusals, and the ptxas budget need no GPU."""
import math

import numpy as np
import pytest

import test_build_resources as res
import test_fp8_blockwise_gpu as bw
import test_fp8_gpu as f8
import test_fp8_grouped_gpu as fg
import test_grouped_gpu as gg
import test_transposed_ops_gpu as tr
from test_transposed_ops_gpu import hooks, sms  # noqa: F401  (fixtures: scheduling hooks reset, SM count)

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")
E4M3, E5M2 = f8.E4M3, f8.E5M2
OUT_F32, OUT_BF16, OUT_F16 = f8.OUT_F32, f8.OUT_BF16, f8.OUT_F16
PAIRS, PAIR_NAME, OUT_NAME = f8.PAIRS, f8.PAIR_NAME, f8.OUT_NAME
OUTS = fg.OUTS
RECIPES, RECIPE_NAME = bw.RECIPES, bw.RECIPE_NAME
B_BLOCKS = (128, 1)                     # a grouped A is always 1 x 128: scale_b 128 x 128 or 1 x 128
ERR_BAD_ARG, ERR_NO_DEVICE, ERR_UNSUPPORTED = fg.ERR_BAD_ARG, fg.ERR_NO_DEVICE, fg.ERR_UNSUPPORTED
MAX_INDEX = bw.MAX_INDEX
cdiv, pad16 = bw.cdiv, fg.pad16


def kernel_name(ta, tb, o, stack):
    return f"tc_{PAIR_NAME[(ta, tb)]}_{OUT_NAME[o]}_{stack}_blk_128x128"


# ==== the C ABI through ctypes (CPU: every refusal happens before the device is touched) =============================
def call_grp(gemm, ta=E4M3, tb=E4M3, total_m=40, n=32, k=32, a=16, lda=None, b=16, ldb=None, stride_b=None, offs=16,
             groups=3, sa=16, sa_row=None, sa_kb=1, sb=16, b_blk=128, sb_kb=None, sb_col=1, ssb=None, c=16, ldc=None,
             out=OUT_BF16):
    """b200_gemm_fp8_blockwise_grouped with raw pointers (16: a dummy aligned non-null pointer, 1: a misaligned one).
    Default scale strides: contiguous (total_m, q) scale_a and (G, q, cols) scale_b."""
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    q, cols = cdiv(k, 128), (cdiv(n, 128) if b_blk == 128 else n)
    sa_row = q if sa_row is None else sa_row
    sb_kb = cols if sb_kb is None else sb_kb
    ssb = q * cols if ssb is None else ssb
    return gemm.lib.b200_gemm_fp8_blockwise_grouped(ta, tb, total_m, n, k, a, lda, b, ldb, stride_b, offs, groups, sa,
                                                    sa_row, sa_kb, sb, b_blk, sb_kb, sb_col, ssb, c, ldc, out, None)


def call_bat(gemm, ta=E4M3, tb=E4M3, m=40, n=32, k=32, a=16, lda=None, stride_a=None, b=16, ldb=None, stride_b=None,
             sa=16, a_blk=1, sa_row=None, sa_kb=1, ssa=None, sb=16, b_blk=128, sb_kb=None, sb_col=1, ssb=None, c=16,
             ldc=None, stride_c=None, batch=3, out=OUT_BF16):
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_a = m * lda if stride_a is None else stride_a
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    stride_c = m * ldc if stride_c is None else stride_c
    q = cdiv(k, 128)
    rows, cols = (m if a_blk == 1 else cdiv(m, 128)), (cdiv(n, 128) if b_blk == 128 else n)
    sa_row = q if sa_row is None else sa_row
    ssa = rows * q if ssa is None else ssa
    sb_kb = cols if sb_kb is None else sb_kb
    ssb = q * cols if ssb is None else ssb
    return gemm.lib.b200_gemm_fp8_blockwise_batched(ta, tb, m, n, k, a, lda, stride_a, b, ldb, stride_b, sa, a_blk, sa_row,
                                                    sa_kb, ssa, sb, b_blk, sb_kb, sb_col, ssb, c, ldc, stride_c, batch,
                                                    out, None)


def test_blockwise_grouped_argument_validation(gemm):
    """Refusals before the device is touched, each at its bound: they hold with or without a GPU."""
    for call in (call_grp, call_bat):
        assert call(gemm, ta=2) == ERR_BAD_ARG and call(gemm, tb=-1) == ERR_BAD_ARG
        assert call(gemm, out=3) == ERR_BAD_ARG and call(gemm, out=-1) == ERR_BAD_ARG
        for bad in (0, 2, 64, 127, 129, -1, -128):
            assert call(gemm, b_blk=bad) == ERR_BAD_ARG
        for kw in ("sa_row", "sa_kb", "sb_kb", "sb_col", "ssb"):
            assert call(gemm, **{kw: -1}) == ERR_BAD_ARG, kw
        assert call(gemm, n=-1) == ERR_BAD_ARG and call(gemm, k=-1) == ERR_BAD_ARG
        assert call(gemm, ta=E5M2, tb=E5M2) == ERR_UNSUPPORTED                     # as b200_gemm_fp8
        assert call(gemm, ldb=31) == ERR_BAD_ARG                                    # B_g is n x k: ldb >= k
        assert call(gemm, lda=31) == ERR_BAD_ARG and call(gemm, ldc=31) == ERR_BAD_ARG
        assert call(gemm, a=None) == ERR_BAD_ARG and call(gemm, b=None) == ERR_BAD_ARG
        assert call(gemm, c=None) == ERR_BAD_ARG
        assert call(gemm, sa=None) == ERR_BAD_ARG and call(gemm, sb=None) == ERR_BAD_ARG
        assert call(gemm, sa=None, k=0, a=None, b=None) == ERR_BAD_ARG              # a null scale with work to do
        assert call(gemm, n=0, a=None, b=None, c=None, sa=None, sb=None) == 0      # no-ops
        # operands the tensor cores cannot read in place
        assert call(gemm, a=1) == ERR_UNSUPPORTED and call(gemm, b=1 + 16) == ERR_UNSUPPORTED
        assert call(gemm, k=24) == ERR_UNSUPPORTED                                  # lda = ldb = 24 bytes
        assert call(gemm, lda=40) == ERR_UNSUPPORTED and call(gemm, ldb=40) == ERR_UNSUPPORTED
        # the last scale index one past the bound (stride 2^59 between the three entries' scale_b: 2^60 in all)
        assert call(gemm, n=2, b_blk=1, sb_kb=0, ssb=1 << 59, sb_col=MAX_INDEX - (1 << 60) + 1) == ERR_BAD_ARG
        assert call(gemm, k=129, sb_kb=MAX_INDEX + 1, ssb=0) == ERR_BAD_ARG
    # grouped: b200_gemm_fp8_grouped's rules
    assert call_grp(gemm, total_m=-1) == ERR_BAD_ARG
    assert call_grp(gemm, groups=-1) == ERR_BAD_ARG and call_grp(gemm, groups=1025) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=-1) == ERR_BAD_ARG
    assert call_grp(gemm, offs=None) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=32 * 32 - 16) == ERR_BAD_ARG                     # B_g overlap
    assert call_grp(gemm, stride_b=0) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=(1 << 60) // 2 + 16) == ERR_BAD_ARG             # (groups - 1) * stride_b > 2^60
    assert call_grp(gemm, ssb=(1 << 60) // 2 + 1) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=32 * 32 + 8) == ERR_UNSUPPORTED                  # not a 16-byte multiple
    assert call_grp(gemm, total_m=1 << 30, n=1 << 20) == ERR_BAD_ARG                # the tile bound
    assert call_grp(gemm, total_m=2, sa_row=MAX_INDEX + 1, sa_kb=0) == ERR_BAD_ARG  # scale_a's last index
    assert call_grp(gemm, total_m=2, k=129, sa_row=0, sa_kb=MAX_INDEX + 1) == ERR_BAD_ARG
    assert call_grp(gemm, groups=0, a=None, b=None, c=None, offs=None, sa=None, sb=None) == 0
    assert call_grp(gemm, total_m=0, a=None, b=None, c=None, offs=None, sa=None, sb=None) == 0
    # batched: b200_gemm_fp8_batched's rules, and b200_gemm_fp8_blockwise's recipes
    for bad in (0, 2, 127, 129, -1):
        assert call_bat(gemm, a_blk=bad) == ERR_BAD_ARG
    assert call_bat(gemm, a_blk=128, b_blk=128) == ERR_UNSUPPORTED                  # not a torch recipe
    assert call_bat(gemm, a_blk=128, b_blk=128, batch=1) == ERR_UNSUPPORTED
    assert call_bat(gemm, m=-1) == ERR_BAD_ARG and call_bat(gemm, batch=-1) == ERR_BAD_ARG
    for kw in ("stride_a", "stride_b", "stride_c", "ssa", "ssb"):
        assert call_bat(gemm, **{kw: -1}) == ERR_BAD_ARG, kw
        assert call_bat(gemm, **{kw: (1 << 60) // 2 + 16}) == ERR_BAD_ARG, kw
    assert call_bat(gemm, stride_c=39 * 32 + 31) == ERR_BAD_ARG                     # entries of C overlap
    assert call_bat(gemm, m=1 << 21, n=1 << 21, batch=3) == ERR_BAD_ARG             # the tile bound
    assert call_bat(gemm, stride_a=40 * 32 - 16) == ERR_UNSUPPORTED                 # overlapping inputs
    assert call_bat(gemm, stride_a=40 * 32 + 8) == ERR_UNSUPPORTED
    assert call_bat(gemm, m=2, sa_kb=0, ssa=1 << 59, sa_row=MAX_INDEX - (1 << 60) + 1) == ERR_BAD_ARG
    assert call_bat(gemm, m=129, a_blk=128, b_blk=1, sa_kb=0, ssa=0, sa_row=MAX_INDEX + 1) == ERR_BAD_ARG
    assert call_bat(gemm, batch=0, a=None, b=None, c=None, sa=None, sb=None) == 0
    assert call_bat(gemm, m=0, a=None, b=None, c=None, sa=None, sb=None) == 0


@pytest.mark.skipif(fg._has_gpu(), reason="checks the no-device behaviour")
def test_blockwise_grouped_accepts_at_the_bounds_without_device(gemm):
    """Legal calls at the bounds reach the device check (-2): every pair, C type and recipe; scale strides of 0; one
    group and 1024 groups; k == 0 with null operands; the last scale index exactly at its bound."""
    for ta, tb in PAIRS:
        for o in OUTS:
            for b_blk in B_BLOCKS:
                assert call_grp(gemm, ta=ta, tb=tb, out=o, b_blk=b_blk) == ERR_NO_DEVICE
            for a_blk, b_blk in RECIPES:
                assert call_bat(gemm, ta=ta, tb=tb, out=o, a_blk=a_blk, b_blk=b_blk) == ERR_NO_DEVICE
    for call in (call_grp, call_bat):
        assert call(gemm, sa_row=0, sa_kb=0, sb_kb=0, sb_col=0, ssb=0) == ERR_NO_DEVICE
        assert call(gemm, k=0, a=None, b=None) == ERR_NO_DEVICE
        assert call(gemm, k=0, a=1, b=1) == ERR_NO_DEVICE                          # k == 0 reads no operand
        assert call(gemm, n=2, b_blk=1, sb_kb=0, ssb=1 << 59, sb_col=MAX_INDEX - (1 << 60)) == ERR_NO_DEVICE
        assert call(gemm, k=129, lda=144, ldb=144, sb_kb=MAX_INDEX, ssb=0) == ERR_NO_DEVICE
    assert call_grp(gemm, groups=1, stride_b=0, ssb=0) == ERR_NO_DEVICE
    assert call_grp(gemm, groups=1024) == ERR_NO_DEVICE
    assert call_grp(gemm, total_m=2, sa_row=MAX_INDEX, sa_kb=0) == ERR_NO_DEVICE
    assert call_bat(gemm, stride_a=0, stride_b=0, ssa=7, ssb=0) == ERR_NO_DEVICE
    assert call_bat(gemm, batch=1, stride_a=0, stride_c=0) == ERR_NO_DEVICE
    assert call_bat(gemm, m=2, sa_kb=0, ssa=1 << 59, sa_row=MAX_INDEX - (1 << 60)) == ERR_NO_DEVICE
    assert call_bat(gemm, m=128, a_blk=128, b_blk=1, sa_kb=0, ssa=0, sa_row=1 << 62) == ERR_NO_DEVICE   # one row block


def test_stacked_blockwise_kernels_do_not_spill():
    """The 18 stacked blockwise kernels (3 pairs x 3 C types x grouped / batch) have 0 spill bytes: the stacked scale
    loader runs in the producer warpgroup's 40 registers."""
    import re
    k = res.kernels()
    names = [n for n in k if "gemm_tc_fp8_kernel" in n and re.search(r"Lb1ELi[12]E", n)]
    assert len(names) == 18, names
    for n in names:
        assert k[n]["spill"] == 0, (n, k[n])


# ==== scaled_grouped_mm: recipe resolution and refusals (CPU) =====================================================
@need_torch
def test_scaled_grouped_mm_resolves_blockwise_shapes(gemm):
    G, T, m, n, k = 3, 300, 200, 300, 401
    q, mb, nb = 4, 2, 3
    ones = torch.ones
    x, xa = fg._fp8((T, k)), fg._fp8((G, m, k))
    B = fg._fp8((G, n, k)).transpose(-2, -1)
    offs = torch.tensor([100, 200, 300], dtype=torch.int32)
    rec = gemm._grouped_blockwise_recipe
    assert rec(x, ones(T, q), ones(G, q, nb), G, n, k) == (1, 128)
    assert rec(x, ones(T, q), ones(G, q, n), G, n, k) == (1, 1)
    assert rec(x, ones(q, T).t(), ones(G, nb, q).transpose(1, 2), G, n, k) == (1, 128)     # strides do not matter
    assert rec(x, ones(cdiv(T, 128), q), ones(G, q, n), G, n, k) is None                   # 128 x 128 A with offs
    assert rec(xa, ones(G, m, q), ones(G, q, nb), G, n, k) == (1, 128)
    assert rec(xa, ones(G, m, q), ones(G, q, n), G, n, k) == (1, 1)
    assert rec(xa, ones(G, mb, q), ones(G, q, n), G, n, k) == (128, 1)
    assert rec(xa, ones(G, mb, q), ones(G, q, nb), G, n, k) is None                        # (128 x 128, 128 x 128)
    # one row / column: two recipes fit, scaled_mm's order decides
    assert rec(fg._fp8((G, 1, k)), ones(G, 1, q), ones(G, q, 1), G, 1, k) == (1, 128)
    sgm = gemm.scaled_grouped_mm
    for A, sa, sb, o in ((x, ones(T, q), ones(G, q, nb), offs), (x, ones(T, q), ones(G, q, n), offs),
                         (xa, ones(G, m, q), ones(G, q, nb), None), (xa, ones(G, m, q), ones(G, q, n), None),
                         (xa, ones(G, mb, q), ones(G, q, n), None)):
        with pytest.raises(ValueError, match="CUDA"):                 # resolved; the CPU tensors are refused next
            sgm(A, B, sa, sb, o)
        with pytest.raises(ValueError, match="use_fast_accum"):
            sgm(A, B, sa, sb, o, use_fast_accum=True)


@need_torch
def test_scaled_grouped_mm_blockwise_refusals(gemm):
    G, T, m, n, k = 3, 300, 200, 300, 401
    q, mb, nb = 4, 2, 3
    ones = torch.ones
    x, xa = fg._fp8((T, k)), fg._fp8((G, m, k))
    B = fg._fp8((G, n, k)).transpose(-2, -1)
    offs = torch.tensor([100, 200, 300], dtype=torch.int32)
    sgm = gemm.scaled_grouped_mm
    bad = [
        (x, ones(T, q + 1), ones(G, q + 1, nb), offs),           # wrong q
        (x, ones(T, q), ones(G, q, nb + 1), offs),               # wrong nb
        (x, ones(T, q), ones(G + 1, q, nb), offs),               # wrong G
        (x, ones(T + 1, q), ones(G, q, nb), offs),
        (x, ones(T, q), ones(q, nb), offs),                      # 2-D scale_b: the rowwise form's shape check
        (x, ones(cdiv(T, 128), q), ones(G, q, n), offs),         # a 128 x 128 A with offs
        (x, ones(T, q).double(), ones(G, q, nb), offs),          # wrong dtype
        (x, ones(T, q), ones(G, q, nb).half(), offs),
        (x, ones(T), ones(G, q, nb), offs),                      # rowwise scale_a with blockwise scale_b
        (xa, ones(G, mb, q), ones(G, q, nb), None),              # (128 x 128, 128 x 128)
        (xa, ones(G, m + 1, q), ones(G, q, n), None),
        (xa, ones(G, m), ones(G, q, nb), None),
        (xa, ones(G, m, q), ones(G, n), None),
    ]
    for A, sa, sb, o in bad:
        with pytest.raises(ValueError):
            sgm(A, B, sa, sb, o)
    with pytest.raises(ValueError):
        sgm(x, B, ones(T, q), ones(G, q, nb))                    # 2-D A needs offs
    with pytest.raises(ValueError, match="use_fast_accum"):
        sgm(x, B, ones(T, q), ones(G, q, nb), offs, use_fast_accum=True)


# ==== GPU: problems with poisoned padding =========================================================================
dev = fg.dev


def nan_padded(vals, pad_last=3, pad_mid=1):
    """vals (..., r, c) as a CUDA view into a NaN-filled buffer with pad_mid NaN rows after each entry's r rows and
    pad_last NaN columns after each row: NaN between the rows and k-blocks of every entry."""
    *lead, r, c = vals.shape
    buf = torch.full(tuple(lead) + (r + pad_mid, c + pad_last), float("nan"), device="cuda")
    view = buf[..., :r, :c]
    view.copy_(dev(vals))
    return view


def make_scales(rng, shape, exact):
    """fp32 block scales: random significands (their products round), or powers of two."""
    if exact:
        return np.exp2(rng.integers(-3, 4, shape)).astype(np.float32)
    return bw.random_scales(rng, shape)


def blockwise_call(gemm, ta, tb, m, n, k, A, lda, B, ldb, Sa, a_blk, Sb, b_blk, C, ldc, o, stream=None):
    """b200_gemm_fp8_blockwise (N, T) with no bias: Sa (rows, q) and Sb (q, cols) passed with their own strides."""
    return gemm.lib.b200_gemm_fp8_blockwise(0, 1, ta, tb, m, n, k, A, lda, B, ldb, Sa.data_ptr(), a_blk,
                                            *bw.strides_of(Sa), Sb.data_ptr(), b_blk, *bw.strides_of(Sb), None, C, ldc,
                                            o, stream)


class Grouped:
    """A grouped blockwise problem: sizes (rows per group) or explicit offs, n, k, B's recipe; operands at padded
    pitches with NaN bytes, scales NaN-fenced between rows and k-blocks.  exact: integer operands in [-2, 2] (every
    block product exact); pow2 (default: exact): power-of-two scales."""

    def __init__(self, ta, tb, sizes, n, k, b_blk, seed, exact=False, pow2=None, offs=None, total_m=None):
        self.ta, self.tb, self.n, self.k, self.b_blk = ta, tb, n, k, b_blk
        self.G = len(sizes) if offs is None else len(offs)
        self.offs_list = list(np.cumsum(sizes)) if offs is None else list(offs)
        self.total_m = total_m if total_m is not None else int(sum(sizes))
        self.ends = gg.clamped_ends(self.offs_list, self.total_m)
        rng = np.random.default_rng(seed)
        self.a8, self.b8, _, _ = fg.operands(rng, ta, tb, self.total_m, n, k, self.G, exact)
        self.A, self.lda, _ = fg.padded(self.a8, pad16(k) + 16)
        self.B, self.ldb, self.stride_b = fg.padded(self.b8, pad16(k) + 32, entry_gap=48)
        q, cols = cdiv(k, 128), (cdiv(n, 128) if b_blk == 128 else n)
        pow2 = exact if pow2 is None else pow2
        self.sa = make_scales(rng, (self.total_m, q), pow2)
        self.sb = make_scales(rng, (self.G, q, cols), pow2)
        self.Sa, self.Sb = nan_padded(self.sa), nan_padded(self.sb)
        self.offs = torch.tensor([int(o) for o in self.offs_list], dtype=torch.int32, device="cuda")
        self.ldc = n + 8

    def c_buf(self, o):
        return torch.full((max(self.total_m, 1), self.ldc), float("nan"), dtype=f8.out_dtype(o), device="cuda")

    def call(self, gemm, C, o, k=None, stream=None, Sa=None, Sb=None):
        Sa = self.Sa if Sa is None else Sa
        Sb = self.Sb if Sb is None else Sb
        return gemm.lib.b200_gemm_fp8_blockwise_grouped(
            self.ta, self.tb, self.total_m, self.n, self.k if k is None else k, self.A.data_ptr(), self.lda,
            self.B.data_ptr(), self.ldb, self.stride_b, self.offs.data_ptr(), self.G, Sa.data_ptr(), Sa.stride(0),
            Sa.stride(1), Sb.data_ptr(), self.b_blk, Sb.stride(1), Sb.stride(2), Sb.stride(0) if self.G > 1 else 0,
            C.data_ptr(), self.ldc, o, stream)

    def reference(self, gemm, o):
        """Each group by b200_gemm_fp8_blockwise (N, T) on contiguous aligned copies of its rows, B_g and scales."""
        C = self.c_buf(o)
        esz = C.element_size()
        lo = 0
        for g, hi in enumerate(self.ends):
            if hi > lo:
                A, lda, _ = fg.padded(self.a8[lo:hi], pad16(self.k))
                B, ldb, _ = fg.padded(self.b8[g], pad16(self.k))
                rc = blockwise_call(gemm, self.ta, self.tb, hi - lo, self.n, self.k, A.data_ptr(), lda, B.data_ptr(), ldb,
                                    dev(self.sa[lo:hi]), 1, dev(self.sb[g]), self.b_blk,
                                    C.data_ptr() + lo * self.ldc * esz, self.ldc, o)
                assert rc == 0, rc
            lo = hi
        torch.cuda.synchronize()
        return C

    def oracle(self, o):
        """The FMA-chain oracle per group, NaN past the last group and past n."""
        want = np.full((max(self.total_m, 1), self.ldc), np.nan, np.float32)
        a = f8.decode(self.a8, self.ta)
        lo = 0
        for g, hi in enumerate(self.ends):
            if hi > lo:
                b = f8.decode(self.b8[g], self.tb).T
                sa_full, sb_full = bw.expand_scales(self.sa[lo:hi], self.sb[g], (1, self.b_blk), hi - lo, self.n)
                want[lo:hi, :self.n] = bw.oracle_blockwise(a[lo:hi], b, sa_full, sb_full, None, o)
            lo = hi
        return want


def run_and_check(gemm, P, o, stack="grp"):
    C = P.c_buf(o)
    assert P.call(gemm, C, o) == 0
    torch.cuda.synchronize()
    assert gemm.last_kernel() == kernel_name(P.ta, P.tb, o, stack)
    return C


# empty groups; groups of 1, 127, 128, 129 and 300 rows; a decreasing offset; the last offset past total_m (clamped)
OFFS_EDGES = ([0, 1, 128, 256, 385, 685, 600, 5000], 760)
# the same kinds of groups, with rows after the last group that must stay NaN
OFFS_TAIL = ([127, 127, 427, 428, 300, 556], 700)


@gpu
@pytest.mark.parametrize("b_blk", B_BLOCKS, ids=["128x128", "1x128"])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_grouped_bit_identical_to_blockwise_per_group(gemm, pair, b_blk):
    """Every C type: each group equals b200_gemm_fp8_blockwise on contiguous copies of its rows, B_g and scales; n is
    not a tile multiple and k is a multiple of 16 but not of 128.  Whole NaN-fenced buffers are compared."""
    ta, tb = pair
    for offs, total_m in (OFFS_EDGES, OFFS_TAIL):
        P = Grouped(ta, tb, None, 200, 400, b_blk, seed=1, offs=offs, total_m=total_m)
        for o in OUTS:
            C = run_and_check(gemm, P, o)
            assert tr.same_bits(C, P.reference(gemm, o)), (offs, o)
            assert bool(torch.isnan(C[P.ends[-1]:]).all()) and bool(torch.isnan(C[:, P.n:]).all())


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_grouped_exact_oracle(gemm, pair):
    """Integer operands and power-of-two scales: every C type and B recipe equals the FMA-chain oracle bit for bit."""
    ta, tb = pair
    for b_blk in B_BLOCKS:
        P = Grouped(ta, tb, [130, 0, 257, 1, 90], 150, 3 * 128 + 16, b_blk, seed=4, exact=True)
        for o in OUTS:
            C = run_and_check(gemm, P, o)
            assert tr.same_bits(C.float().cpu(), torch.from_numpy(P.oracle(o))), (b_blk, o)


@gpu
def test_grouped_random_scales_match_the_oracle(gemm):
    """Integer operands with random-significand scales pin rn(sa * sb) and the FMA order: still the oracle's bits."""
    for b_blk in B_BLOCKS:
        P = Grouped(E4M3, E4M3, [200, 3, 0, 129], 260, 700, b_blk, seed=5, exact=True, pow2=False)
        C = run_and_check(gemm, P, OUT_F32)
        assert tr.same_bits(C.cpu(), torch.from_numpy(P.oracle(OUT_F32))), b_blk


@gpu
def test_grouped_scale_layouts_are_bit_identical(gemm):
    """Outer-dim-major, row-major and padded scale layouts give the same bits; a scale_b broadcast across groups
    (stride 0) equals the materialised copy."""
    for b_blk in B_BLOCKS:
        P = Grouped(E4M3, E5M2, [300, 45, 129], 200, 520, b_blk, seed=7)
        ref = run_and_check(gemm, P, OUT_F32)
        sa_views = [dev(P.sa), dev(np.ascontiguousarray(P.sa.T)).t(), P.Sa]
        sb_views = [dev(P.sb), dev(np.ascontiguousarray(P.sb.transpose(0, 2, 1))).transpose(1, 2), P.Sb]
        for Sa in sa_views:
            for Sb in sb_views:
                C = P.c_buf(OUT_F32)
                assert P.call(gemm, C, OUT_F32, Sa=Sa, Sb=Sb) == 0
                torch.cuda.synchronize()
                assert tr.same_bits(C, ref), (Sa.stride(), Sb.stride())
        Sb0 = dev(P.sb[:1]).expand(P.sb.shape)
        assert Sb0.stride(0) == 0
        C = P.c_buf(OUT_F32)
        assert P.call(gemm, C, OUT_F32, Sb=Sb0) == 0
        P.sb = np.ascontiguousarray(np.broadcast_to(P.sb[:1], P.sb.shape))
        torch.cuda.synchronize()
        assert tr.same_bits(C, P.reference(gemm, OUT_F32)), b_blk


@gpu
@pytest.mark.parametrize("k", [16, 112, 128, 144, 1040])
def test_grouped_k_tails(gemm, k):
    """k below, at and past one k-block, a partial last k-block, n not a multiple of 128."""
    for b_blk in B_BLOCKS:
        P = Grouped(E4M3, E4M3, [1, 127, 128, 129, 0, 300], 200, k, b_blk, seed=k)
        for o in (OUT_F32, OUT_BF16):
            C = run_and_check(gemm, P, o)
            assert tr.same_bits(C, P.reference(gemm, o)), (b_blk, o)


@gpu
def test_grouped_k_zero(gemm):
    """k == 0: +0 over rows [0, end_{G-1}) through fill_zero_grp, no scale read (NaN scales), rows after the last group
    and columns past n untouched."""
    P = Grouped(E4M3, E4M3, None, 64, 32, 128, seed=8, offs=[40, 40, 140], total_m=160)
    P.Sa.fill_(float("nan"))
    P.Sb.fill_(float("nan"))
    for o in OUTS:
        C = P.c_buf(o)
        assert P.call(gemm, C, o, k=0) == 0
        torch.cuda.synchronize()
        assert gemm.last_kernel() == "fill_zero_grp"
        assert bool((C[:140, :64].float() == 0).all()) and not bool(torch.signbit(C[:140, :64].float()).any())
        assert bool(torch.isnan(C[140:]).all()) and bool(torch.isnan(C[:, 64:]).all())


@gpu
def test_many_groups(gemm):
    """256 groups with Zipf sizes, and a call with 1024 groups (most of them empty)."""
    rng = np.random.default_rng(9)
    zipf = np.minimum(rng.zipf(1.5, 256), 400)
    zipf[rng.choice(256, 40, replace=False)] = 0
    P = Grouped(E4M3, E4M3, list(zipf), 136, 272, 128, seed=10)
    C = run_and_check(gemm, P, OUT_BF16)
    assert tr.same_bits(C, P.reference(gemm, OUT_BF16))
    sizes = np.zeros(1024, np.int64)
    sizes[rng.choice(1024, 60, replace=False)] = rng.integers(1, 90, 60)
    P = Grouped(E4M3, E4M3, list(sizes), 64, 144, 1, seed=11)
    C = run_and_check(gemm, P, OUT_F32)
    assert tr.same_bits(C, P.reference(gemm, OUT_F32))


@gpu
def test_cuda_graph_replay_with_new_offsets_and_scales(gemm):
    """One captured grouped call (a host synchronisation inside it would fail the capture); offs and both scales are
    rewritten in place on the device between replays, and each replay equals the eager call on the new values."""
    P = Grouped(E4M3, E4M3, [125] * 8, 256, 3 * 128 + 64, 128, seed=12)
    C = P.c_buf(OUT_BF16)
    assert P.call(gemm, C, OUT_BF16) == 0                             # tensor maps and kernel attributes set up first
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert P.call(gemm, C, OUT_BF16, stream=torch.cuda.current_stream().cuda_stream) == 0
    rng = np.random.default_rng(13)
    for offs in ([600, 600, 700, 700, 900, 990, 1000, 1000], [0, 10, 20, 30, 40, 50, 60, 900]):
        C.fill_(float("nan"))
        P.offs.copy_(torch.tensor(offs, dtype=torch.int32))
        P.Sa.copy_(torch.from_numpy(bw.random_scales(rng, tuple(P.Sa.shape))))
        P.Sb.copy_(torch.from_numpy(bw.random_scales(rng, tuple(P.Sb.shape))))
        graph.replay()
        torch.cuda.synchronize()
        eager = P.c_buf(OUT_BF16)
        assert P.call(gemm, eager, OUT_BF16) == 0
        torch.cuda.synchronize()
        assert tr.same_bits(C, eager), offs
        P.ends = gg.clamped_ends(offs, P.total_m)
        P.sa, P.sb = P.Sa.cpu().numpy(), P.Sb.cpu().numpy()
        assert tr.same_bits(C, P.reference(gemm, OUT_BF16)), offs
        assert bool(torch.isnan(C[P.ends[-1]:]).all())


# ==== batched ======================================================================================================
class Batched:
    def __init__(self, ta, tb, batch, m, n, k, blocks, seed, broadcast_a=False):
        self.ta, self.tb, self.batch, self.m, self.n, self.k, self.blocks = ta, tb, batch, m, n, k, blocks
        rng = np.random.default_rng(seed)
        a8, self.b8, _, _ = fg.operands(rng, ta, tb, m, n, k, batch, False)
        self.a8 = np.broadcast_to(a8, (batch, m, k)) if broadcast_a else \
            fg.operands(rng, ta, tb, batch * m, 1, k, 1, False)[0].reshape(batch, m, k)
        self.A, self.lda, self.stride_a = fg.padded(a8 if broadcast_a else self.a8, pad16(k) + 16, entry_gap=32)
        if broadcast_a:
            self.stride_a = 0
        self.B, self.ldb, self.stride_b = fg.padded(self.b8, pad16(k), entry_gap=16)
        q = cdiv(k, 128)
        rows = m if blocks[0] == 1 else cdiv(m, 128)
        cols = n if blocks[1] == 1 else cdiv(n, 128)
        self.sa = bw.random_scales(rng, (batch, rows, q))
        self.sb = bw.random_scales(rng, (batch, q, cols))
        self.Sa, self.Sb = nan_padded(self.sa), nan_padded(self.sb)
        self.ldc = n + 8
        self.stride_c = (m + 1) * self.ldc

    def c_buf(self, o):
        return torch.full((self.batch * (self.m + 1), self.ldc), float("nan"), dtype=f8.out_dtype(o), device="cuda")

    def call(self, gemm, C, o, k=None):
        Sa, Sb = self.Sa, self.Sb
        return gemm.lib.b200_gemm_fp8_blockwise_batched(
            self.ta, self.tb, self.m, self.n, self.k if k is None else k, self.A.data_ptr(), self.lda, self.stride_a,
            self.B.data_ptr(), self.ldb, self.stride_b, Sa.data_ptr(), self.blocks[0], Sa.stride(1), Sa.stride(2),
            Sa.stride(0), Sb.data_ptr(), self.blocks[1], Sb.stride(1), Sb.stride(2), Sb.stride(0), C.data_ptr(),
            self.ldc, self.stride_c, self.batch, o, None)

    def reference(self, gemm, o):
        C = self.c_buf(o)
        esz = C.element_size()
        for e in range(self.batch):
            A, lda, _ = fg.padded(np.ascontiguousarray(self.a8[e]), pad16(self.k))
            B, ldb, _ = fg.padded(self.b8[e], pad16(self.k))
            rc = blockwise_call(gemm, self.ta, self.tb, self.m, self.n, self.k, A.data_ptr(), lda, B.data_ptr(), ldb,
                                dev(self.sa[e]), self.blocks[0], dev(self.sb[e]), self.blocks[1],
                                C.data_ptr() + e * self.stride_c * esz, self.ldc, o)
            assert rc == 0, rc
        torch.cuda.synchronize()
        return C


@gpu
@pytest.mark.parametrize("blocks", RECIPES, ids=lambda b: RECIPE_NAME[b])
@pytest.mark.parametrize("broadcast_a", [False, True], ids=["strided", "broadcast-A"])
def test_batched_bit_identical_to_blockwise_per_entry(gemm, blocks, broadcast_a):
    """Every pair and C type: each entry equals its own b200_gemm_fp8_blockwise call, with a broadcast A (stride 0)
    scaled by each entry's own scale_a; the gap rows between entries of C stay NaN."""
    for ta, tb in PAIRS:
        P = Batched(ta, tb, 4, 300, 200, 464, blocks, seed=14, broadcast_a=broadcast_a)
        for o in OUTS:
            C = P.c_buf(o)
            assert P.call(gemm, C, o) == 0
            torch.cuda.synchronize()
            assert gemm.last_kernel() == kernel_name(ta, tb, o, "bat")
            assert tr.same_bits(C, P.reference(gemm, o)), (ta, tb, o)


@gpu
def test_batch_of_one_is_the_blockwise_call(gemm):
    """batch == 1 is the (N, T) b200_gemm_fp8_blockwise call: same kernel name and bits; k == 0 of a batch is
    fill_zero_bat."""
    for blocks in RECIPES:
        P = Batched(E4M3, E4M3, 1, 300, 200, 208, blocks, seed=15)
        C = P.c_buf(OUT_BF16)
        assert P.call(gemm, C, OUT_BF16) == 0
        assert gemm.last_kernel() == "tc_e4m3_obf16_blk_128x128"
        assert tr.same_bits(C, P.reference(gemm, OUT_BF16)), blocks
    Q = Batched(E4M3, E4M3, 3, 20, 40, 32, (1, 128), seed=16)
    Q.Sa.fill_(float("nan"))
    C = Q.c_buf(OUT_F32)
    assert Q.call(gemm, C, OUT_F32, k=0) == 0
    torch.cuda.synchronize()
    assert gemm.last_kernel() == "fill_zero_bat"
    for e in range(3):
        blk = C[e * 21:e * 21 + 21]
        assert bool((blk[:20, :40] == 0).all()) and bool(torch.isnan(blk[20]).all()) and bool(torch.isnan(blk[:, 40:]).all())


# ==== scaled_grouped_mm end to end, and a DeepSeek-V3-shaped layer =================================================
def quantise_1x128(x):
    """e4m3 per 1 x 128 group along the last dimension (amax / 448): q, scales (..., rows, k / 128)."""
    *lead, r, k = x.shape
    g = x.reshape(*lead, r, k // 128, 128)
    s = (g.abs().amax(dim=-1) / 448).clamp_min(1e-12)
    return (g / s[..., None]).reshape(x.shape).to(torch.float8_e4m3fn), s


def quantise_128x128(w):
    """e4m3 per 128 x 128 block of each (n, k) weight: q, scales (G, n / 128, k / 128)."""
    G, n, k = w.shape
    g = w.reshape(G, n // 128, 128, k // 128, 128)
    s = (g.abs().amax(dim=(2, 4)) / 448).clamp_min(1e-12)
    return (g / s[:, :, None, :, None]).reshape(w.shape).to(torch.float8_e4m3fn), s


@gpu
def test_scaled_grouped_mm_blockwise_end_to_end(gemm):
    """scaled_grouped_mm with torch's outer-dim-major scales equals the ABI call on the same tensors, for the grouped
    and the batched form and each recipe."""
    rng = np.random.default_rng(17)
    G, n, k = 4, 256, 512
    q = k // 128
    P = Grouped(E4M3, E4M3, [100, 0, 300, 57], n, k, 128, seed=18)
    xu8 = P.A[:P.total_m * P.lda].view(P.total_m, P.lda)[:, :k]          # the padded rows, read in place
    x = xu8.view(torch.float8_e4m3fn)
    W = dev(P.b8).view(torch.float8_e4m3fn)                              # (G, n, k)
    Sa = dev(np.ascontiguousarray(P.sa.T)).t()
    for b_blk in B_BLOCKS:
        sb = bw.random_scales(rng, (G, q, n // 128 if b_blk == 128 else n))
        y = gemm.scaled_grouped_mm(x, W.transpose(-2, -1), Sa, dev(sb), P.offs, out_dtype=torch.float32)
        assert gemm.last_kernel() == "tc_e4m3_of32_grp_blk_128x128"
        P.sa, P.sb, P.b_blk = Sa.cpu().numpy(), sb, b_blk
        want = P.reference(gemm, OUT_F32)[:, :n]
        assert tr.same_bits(y[:P.ends[-1]], want[:P.ends[-1]]), b_blk
    xa = torch.stack([xu8[:200]] * G).view(torch.float8_e4m3fn)
    for blocks in RECIPES:
        rows = 200 if blocks[0] == 1 else 2
        sa = bw.random_scales(rng, (G, rows, q))
        sb = bw.random_scales(rng, (G, q, n if blocks[1] == 1 else n // 128))
        y = gemm.scaled_grouped_mm(xa, W.transpose(-2, -1), dev(sa), dev(sb), out_dtype=torch.bfloat16)
        assert gemm.last_kernel() == "tc_e4m3_obf16_bat_blk_128x128"
        for g in range(G):
            ref = torch.empty((200, n), dtype=torch.bfloat16, device="cuda")
            assert blockwise_call(gemm, E4M3, E4M3, 200, n, k, xa[g].data_ptr(), xa.stride(1), W[g].data_ptr(), k,
                                  dev(sa[g]), blocks[0], dev(sb[g]), blocks[1], ref.data_ptr(), n, OUT_BF16) == 0
            torch.cuda.synchronize()
            assert tr.same_bits(y[g], ref), (blocks, g)


@gpu
def test_deepseek_v3_shaped_layer(gemm):
    """An MoE up projection quantised as DeepSeek-V3 does (x per 1 x 128, each expert's W per 128 x 128): fp32 out
    within rel_bound(k) of the float64 dequantised product, bf16 within that plus one bf16 rounding."""
    torch.manual_seed(19)
    G, d, dff = 8, 2048, 1024
    sizes = [700, 40, 0, 513, 300, 1, 900, 94]
    offs = torch.tensor(np.cumsum(sizes), dtype=torch.int32, device="cuda")
    x = torch.randn((sum(sizes), d), device="cuda")
    W = torch.randn((G, dff, d), device="cuda") * 0.02
    xq, sx = quantise_1x128(x)                                 # (T, d / 128)
    wq, sw = quantise_128x128(W)                               # (G, dff / 128, d / 128)
    scale_a = sx.t().contiguous().t()                          # outer-dim-major, as torch takes it
    scale_b = sw.transpose(1, 2)                               # (G, q, dff / 128)
    y32 = gemm.scaled_grouped_mm(xq, wq.transpose(-2, -1), scale_a, scale_b, offs, out_dtype=torch.float32)
    assert gemm.last_kernel() == "tc_e4m3_of32_grp_blk_128x128"
    y16 = gemm.scaled_grouped_mm(xq, wq.transpose(-2, -1), scale_a, scale_b, offs)
    assert y16.dtype == torch.bfloat16 and gemm.last_kernel() == "tc_e4m3_obf16_grp_blk_128x128"
    ends = [0] + offs.tolist()
    for g in range(G):
        lo, hi = ends[g], ends[g + 1]
        if hi == lo:
            continue
        rows = torch.arange(lo, hi, 7, device="cuda")
        a = xq[rows].float().cpu().numpy()
        b = wq[g].float().cpu().numpy().T
        sa_full = sx[rows].cpu().numpy()
        sb_full = np.repeat(sw[g].t().cpu().numpy(), 128, axis=1)
        ex, w = bw.exact_and_weight(a, b, sa_full, sb_full)
        err32 = np.abs(y32[rows].double().cpu().numpy() - ex)
        assert bool((err32 <= bw.rel_bound(d) * w).all()), (g, float((err32 / w).max()))
        err16 = np.abs(y16[rows].double().cpu().numpy() - ex)
        assert bool((err16 <= bw.rel_bound(d) * w + 2.0 ** -8 * np.abs(ex)).all()), g
    assert math.isfinite(float(y32[:ends[-1]].abs().max()))
