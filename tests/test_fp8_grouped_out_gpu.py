"""FP8 outputs of the grouped and batched FP8 GEMMs (b200_gemm_fp8_grouped_q8, _batched_q8, _blockwise_grouped_q8,
_blockwise_batched_q8) and scaled_grouped_mm_quant().

Every group or entry's C and scale_c must be bit for bit the single-matrix dynamic-mode call on that entry's rows, B
and scales, (N, T), null bias and null scale_result: b200_gemm_fp8_q8 for rowwise scales at the same tile width,
b200_gemm_fp8_blockwise_q8 for blockwise scales.  The stacked calls run on NaN-padded operands and NaN-fenced scales;
C and scale_c sit in sentinel-filled buffers, so rows past the last group and bytes past n or ldc are checked
untouched.  On integer operands with power-of-two scales the result is also the numpy quantisation (quant_dynamic) of
the exact fp32 oracle.

The argument checks, the kernel table, the ptxas resources and the Python refusals need no GPU."""
import re

import numpy as np
import pytest

import test_build_resources as res
import test_fp8_blockwise_gpu as bw
import test_fp8_blockwise_grouped_gpu as bg
import test_fp8_gpu as f8
import test_fp8_grouped_gpu as fg
import test_fp8_out_gpu as fo
import test_grouped_gpu as gg
from test_transposed_ops_gpu import hooks, sms  # noqa: F401  (fixtures: scheduling hooks reset, SM count)

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")
E4M3, E5M2, OP_N, OP_T = f8.E4M3, f8.E5M2, f8.OP_N, f8.OP_T
PAIRS, PAIR_NAME, CT_NAME = f8.PAIRS, f8.PAIR_NAME, fo.CT_NAME
ERR_BAD_ARG, ERR_NO_DEVICE, ERR_UNSUPPORTED = fg.ERR_BAD_ARG, fg.ERR_NO_DEVICE, fg.ERR_UNSUPPORTED
ACTS = (fo.ACT_NONE, fo.ACT_RELU, fo.ACT_GELU, fo.ACT_GELU_TANH)
MAX_INDEX = bw.MAX_INDEX
SC_SENTINEL = fo.SC_SENTINEL
cdiv, pad16 = bw.cdiv, fg.pad16
C_FENCE = 0xA5                          # C's fence byte: not a byte any quantised value of these tests takes past n

# Input recipes: ("row", mode) with mode "acc" (promoted) or a forced fast width 256 / 128; ("blk", (a_blk, b_blk)).
GROUPED_RECIPES = [("row", "acc"), ("row", 256), ("row", 128), ("blk", (1, 128)), ("blk", (1, 1))]
BATCHED_RECIPES = [("row", "acc"), ("row", 256), ("row", 128)] + [("blk", b) for b in bw.RECIPES]
RECIPE_ID = lambda r: f"{r[0]}-{r[1]}" if r[0] == "row" else "blk-" + bw.RECIPE_NAME[r[1]]  # noqa: E731


def kernel_name(ta, tb, ct, stack, recipe):
    if recipe[0] == "blk":
        width = "blk_128x128"
    else:
        width = "acc_128x128" if recipe[1] == "acc" else f"128x{recipe[1]}"
    return f"tc_{PAIR_NAME[(ta, tb)]}_{CT_NAME[ct]}_{stack}_{width}"


def case_table():
    """(pair, ct, stack, recipe) of the GPU bit-identity cases; together they reach every new kernel."""
    for pair in PAIRS:
        for ct in (E4M3, E5M2):
            for stack, recipes in (("grp", GROUPED_RECIPES), ("bat", BATCHED_RECIPES)):
                for recipe in recipes:
                    yield pair, ct, stack, recipe


def test_case_table_reaches_every_new_kernel():
    want = {f"tc_{PAIR_NAME[p]}_{CT_NAME[ct]}_{s}_{w}" for p in PAIRS for ct in (E4M3, E5M2) for s in ("grp", "bat")
            for w in ("128x256", "128x128", "acc_128x128", "blk_128x128")}
    assert len(want) == 48
    assert {kernel_name(*pair, ct, stack, recipe) for pair, ct, stack, recipe in case_table()} == want


def test_stacked_fp8_output_kernels_do_not_spill():
    """48 gemm_tc_fp8_q8_stacked_kernel instantiations (3 pairs x 2 C types x {256, 128, promoted, blockwise} x
    {grouped, batch}) and the 4 k == 0 kernels, all with 0 spill bytes; none of them is a gemm_tc_fp8_kernel."""
    k = res.kernels()
    names = [n for n in k if "gemm_tc_fp8_q8_stacked_kernel" in n]
    assert len(names) == 48, names
    assert len([n for n in names if re.search(r"Lb1ELi[12]E", n)]) == 12
    k0 = [n for n in k if "fp8_q8_k0_stacked_kernel" in n]
    assert len(k0) == 4, k0
    for n in names + k0:
        assert k[n]["spill"] == 0, (n, k[n])
        assert "gemm_tc_fp8_kernel" not in n


# ==== the C ABI through ctypes (CPU: every refusal happens before the device is touched) =============================
def call_grp(gemm, ta=E4M3, tb=E4M3, total_m=40, n=32, k=32, a=16, lda=None, b=16, ldb=None, stride_b=None, offs=16,
             groups=3, sa=16, sb=16, ssb=32, act=0, fast=0, ct=E4M3, c=16, ldc=None, sc=16, sc_row=None, sc_blk=1):
    """b200_gemm_fp8_grouped_q8 with raw pointers (16: a dummy aligned non-null pointer, 1: a misaligned one)."""
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    sc_row = cdiv(n, 128) if sc_row is None else sc_row
    return gemm.lib.b200_gemm_fp8_grouped_q8(ta, tb, total_m, n, k, a, lda, b, ldb, stride_b, offs, groups, sa, sb, ssb,
                                             act, fast, ct, c, ldc, sc, sc_row, sc_blk, None)


def call_bat(gemm, ta=E4M3, tb=E4M3, m=40, n=32, k=32, a=16, lda=None, stride_a=None, b=16, ldb=None, stride_b=None,
             sa=16, ssa=40, sb=16, ssb=32, act=0, fast=0, ct=E4M3, c=16, ldc=None, stride_c=None, sc=16, sc_row=None,
             sc_blk=1, sc_e=None, batch=3):
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_a = m * lda if stride_a is None else stride_a
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    stride_c = m * ldc if stride_c is None else stride_c
    sc_row = cdiv(n, 128) if sc_row is None else sc_row
    sc_e = m * cdiv(n, 128) if sc_e is None else sc_e
    return gemm.lib.b200_gemm_fp8_batched_q8(ta, tb, m, n, k, a, lda, stride_a, b, ldb, stride_b, sa, ssa, sb, ssb, act,
                                             fast, ct, c, ldc, stride_c, sc, sc_row, sc_blk, sc_e, batch, None)


def call_bgrp(gemm, ta=E4M3, tb=E4M3, total_m=40, n=32, k=32, a=16, lda=None, b=16, ldb=None, stride_b=None, offs=16,
              groups=3, sa=16, sa_row=None, sa_kb=1, sb=16, b_blk=128, sb_kb=None, sb_col=1, ssb=None, act=0, fast=0,
              ct=E4M3, c=16, ldc=None, sc=16, sc_row=None, sc_blk=1):
    assert fast == 0
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    q, cols = cdiv(k, 128), (cdiv(n, 128) if b_blk == 128 else n)
    sa_row = q if sa_row is None else sa_row
    sb_kb = cols if sb_kb is None else sb_kb
    ssb = q * cols if ssb is None else ssb
    sc_row = cdiv(n, 128) if sc_row is None else sc_row
    return gemm.lib.b200_gemm_fp8_blockwise_grouped_q8(ta, tb, total_m, n, k, a, lda, b, ldb, stride_b, offs, groups, sa,
                                                       sa_row, sa_kb, sb, b_blk, sb_kb, sb_col, ssb, act, ct, c, ldc, sc,
                                                       sc_row, sc_blk, None)


def call_bbat(gemm, ta=E4M3, tb=E4M3, m=40, n=32, k=32, a=16, lda=None, stride_a=None, b=16, ldb=None, stride_b=None,
              sa=16, a_blk=1, sa_row=None, sa_kb=1, ssa=None, sb=16, b_blk=128, sb_kb=None, sb_col=1, ssb=None, act=0,
              fast=0, ct=E4M3, c=16, ldc=None, stride_c=None, sc=16, sc_row=None, sc_blk=1, sc_e=None, batch=3):
    assert fast == 0
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
    sc_row = cdiv(n, 128) if sc_row is None else sc_row
    sc_e = m * cdiv(n, 128) if sc_e is None else sc_e
    return gemm.lib.b200_gemm_fp8_blockwise_batched_q8(ta, tb, m, n, k, a, lda, stride_a, b, ldb, stride_b, sa, a_blk,
                                                       sa_row, sa_kb, ssa, sb, b_blk, sb_kb, sb_col, ssb, act, ct, c, ldc,
                                                       stride_c, sc, sc_row, sc_blk, sc_e, batch, None)


CALLS = (call_grp, call_bat, call_bgrp, call_bbat)
GROUPED_CALLS, BATCHED_CALLS = (call_grp, call_bgrp), (call_bat, call_bbat)
SIZE = {call_grp: "total_m", call_bgrp: "total_m", call_bat: "m", call_bbat: "m"}


def test_grouped_q8_argument_validation(gemm):
    """Refusals before the device is touched, each at its bound: they hold with or without a GPU."""
    for call in CALLS:
        rows = SIZE[call]
        # the output arguments (fp8_check's first checks)
        assert call(gemm, ct=2) == ERR_BAD_ARG and call(gemm, ct=-1) == ERR_BAD_ARG
        assert call(gemm, act=4) == ERR_BAD_ARG and call(gemm, act=-1) == ERR_BAD_ARG
        assert call(gemm, sc_row=-1) == ERR_BAD_ARG and call(gemm, sc_blk=-1) == ERR_BAD_ARG
        assert call(gemm, sc=None) == ERR_BAD_ARG                                   # null scale_c with work to do
        assert call(gemm, n=0, ct=2) == ERR_BAD_ARG                                  # before the no-op
        # scale_c layouts that could overlap (4 rows, n = 300: q_n = 3)
        for sc_row, sc_blk in ((2, 1), (3, 0), (1, 3), (0, 4), (3, 3), (4, 2)):
            assert call(gemm, **{rows: 4}, n=300, sc_row=sc_row, sc_blk=sc_blk, sc_e=64) == ERR_BAD_ARG \
                if call in BATCHED_CALLS else call(gemm, **{rows: 4}, n=300, sc_row=sc_row, sc_blk=sc_blk) == ERR_BAD_ARG
        # the last scale index past the bound
        assert call(gemm, **{rows: 4}, n=300, sc_row=MAX_INDEX, sc_blk=1) == ERR_BAD_ARG
        # inherited from the parents
        assert call(gemm, ta=2) == ERR_BAD_ARG and call(gemm, tb=-1) == ERR_BAD_ARG
        assert call(gemm, ta=E5M2, tb=E5M2) == ERR_UNSUPPORTED
        assert call(gemm, n=-1) == ERR_BAD_ARG and call(gemm, k=-1) == ERR_BAD_ARG
        assert call(gemm, lda=31) == ERR_BAD_ARG and call(gemm, ldb=31) == ERR_BAD_ARG and call(gemm, ldc=31) == ERR_BAD_ARG
        assert call(gemm, a=None) == ERR_BAD_ARG and call(gemm, c=None) == ERR_BAD_ARG and call(gemm, sa=None) == ERR_BAD_ARG
        assert call(gemm, a=1) == ERR_UNSUPPORTED                                    # not read in place
        # nothing to do: a no-op whatever the scale pointers
        assert call(gemm, n=0, sc=None, a=None, b=None, c=None, sa=None, sb=None) == 0
        assert call(gemm, **{rows: 0}, sc=None, a=None, b=None, c=None, sa=None, sb=None) == 0
    for call in GROUPED_CALLS:
        assert call(gemm, groups=1025) == ERR_BAD_ARG and call(gemm, offs=None) == ERR_BAD_ARG
        assert call(gemm, groups=0, sc=None, a=None, b=None, c=None, offs=None) == 0
        assert call(gemm, stride_b=32 * 32 - 1) == ERR_BAD_ARG                      # B_g would overlap
    for call in BATCHED_CALLS:
        assert call(gemm, batch=-1) == ERR_BAD_ARG and call(gemm, sc_e=-1) == ERR_BAD_ARG
        assert call(gemm, batch=0, sc=None, a=None, b=None, c=None) == 0
        assert call(gemm, stride_c=39 * 32 + 31) == ERR_BAD_ARG                      # entries of C would overlap
        # entries of scale_c: one entry's last index + 1 apart at least (40 rows, q_n = 1: 40), both layouts
        assert call(gemm, sc_e=39) == ERR_BAD_ARG
        assert call(gemm, n=300, sc_row=1, sc_blk=40, sc_e=119) == ERR_BAD_ARG       # outer-dim-major: 2 * 40 + 39 + 1
        # sc_entry_stride bounded like the other entry strides: (batch - 1) * stride <= 2^60
        assert call(gemm, sc_e=(1 << 59) + 1) == ERR_BAD_ARG
        assert call(gemm, m=1, n=200, sc_row=1, sc_blk=(1 << 60), sc_e=1 << 60, batch=2) == ERR_BAD_ARG  # overlap
    assert call_grp(gemm, fast=2) == ERR_BAD_ARG and call_bat(gemm, fast=-1) == ERR_BAD_ARG
    assert call_bgrp(gemm, b_blk=2) == ERR_BAD_ARG and call_bbat(gemm, a_blk=128, b_blk=128) == ERR_UNSUPPORTED
    assert call_bgrp(gemm, total_m=2, sa_kb=0, sa_row=MAX_INDEX + 1) == ERR_BAD_ARG   # the parent's scale_a bound


@pytest.mark.skipif(fg._has_gpu(), reason="checks the no-device behaviour")
def test_grouped_q8_accepts_at_the_bounds_without_device(gemm):
    """Legal calls at the bounds reach the device check (-2)."""
    for call in CALLS:
        rows = SIZE[call]
        for ct in (E4M3, E5M2):
            for act in ACTS:
                assert call(gemm, ct=ct, act=act) == ERR_NO_DEVICE
        for ta, tb in PAIRS:
            assert call(gemm, ta=ta, tb=tb) == ERR_NO_DEVICE
        # both layouts, packed and padded (4 rows, q_n = 3; a batch's entries 12 apart: the last index is 11)
        for sc_row, sc_blk in ((3, 1), (9, 1), (1, 4), (1, 9)):
            last = 3 * sc_row + 2 * sc_blk
            assert call(gemm, **{rows: 4}, n=300, sc_row=sc_row, sc_blk=sc_blk, **(
                {"sc_e": last + 1} if call in BATCHED_CALLS else {})) == ERR_NO_DEVICE, (call, sc_row, sc_blk)
        assert call(gemm, **{rows: 1}, n=300, sc_row=0, sc_blk=1, **(
            {"sc_e": 3} if call in BATCHED_CALLS else {})) == ERR_NO_DEVICE          # extent-1 rows: the row stride is free
        assert call(gemm, **{rows: 4}, n=100, sc_row=1, sc_blk=0) == ERR_NO_DEVICE  # one block: the block stride is free
        assert call(gemm, k=0, a=None, b=None) == ERR_NO_DEVICE                       # k == 0 still writes C and scale_c
        if call in GROUPED_CALLS:
            assert call(gemm, total_m=2, n=300, sc_row=(MAX_INDEX - 2), sc_blk=1) == ERR_NO_DEVICE
            assert call(gemm, groups=1024) == ERR_NO_DEVICE
    for call in BATCHED_CALLS:
        assert call(gemm, sc_e=40) == ERR_NO_DEVICE                                   # exactly one entry apart
        assert call(gemm, n=300, sc_row=1, sc_blk=40, sc_e=120) == ERR_NO_DEVICE
        assert call(gemm, sc_e=1 << 59) == ERR_NO_DEVICE                              # (batch - 1) * stride = 2^60
        # entries 2^60 apart, each's last index 2^60 - 1: the last index, entry term included, is INT64_MAX / 4
        assert call(gemm, m=1, n=200, sc_row=1, sc_blk=(1 << 60) - 1, sc_e=1 << 60, batch=2) == ERR_NO_DEVICE
        assert call(gemm, batch=1, sc_e=0, stride_a=0, stride_c=0) == ERR_NO_DEVICE   # the single-matrix call
        assert call(gemm, stride_a=0) == ERR_NO_DEVICE                                # a broadcast A
    for fast in (0, 1):
        assert call_grp(gemm, fast=fast) == ERR_NO_DEVICE and call_bat(gemm, fast=fast) == ERR_NO_DEVICE
    for b_blk in (1, 128):
        assert call_bgrp(gemm, b_blk=b_blk) == ERR_NO_DEVICE
    for a_blk, b_blk in bw.RECIPES:
        assert call_bbat(gemm, a_blk=a_blk, b_blk=b_blk) == ERR_NO_DEVICE


# ==== scaled_grouped_mm_quant: resolution and refusals (CPU) ======================================================
def _fp8(shape, t=E4M3):
    return torch.zeros(shape, dtype=torch.float32).to(f8.fp8_dtype(t))


@need_torch
def test_scaled_grouped_mm_quant_resolution_and_refusals(gemm):
    G, T, m, n, k = 3, 300, 200, 300, 401
    q, nb = cdiv(k, 128), cdiv(n, 128)
    sq = gemm.scaled_grouped_mm_quant
    x, x3 = _fp8((T, k)), _fp8((G, m, k))
    W = _fp8((G, n, k)).transpose(-2, -1)                               # (G, k, n), column-major per group
    offs = torch.tensor([100, 200, 300], dtype=torch.int32)
    row_grp = (torch.ones(T), torch.ones(G, n))
    row_bat = (torch.ones(G, m), torch.ones(G, n))
    blk_grp = [(torch.ones(T, q), torch.ones(G, q, c)) for c in (nb, n)]
    blk_bat = [(torch.ones(G, r, q), torch.ones(G, q, c)) for r, c in ((m, nb), (m, n), (cdiv(m, 128), n))]
    # every recipe resolves and reaches the CUDA check, with both C types and every activation
    for A, o, scales in [(x, offs, row_grp)] + [(x, offs, s) for s in blk_grp] + [(x3, None, row_bat)] + \
                        [(x3, None, s) for s in blk_bat]:
        for dt in (None, torch.float8_e4m3fn, torch.float8_e5m2):
            for act in (None, "relu", "gelu", "gelu_tanh"):
                with pytest.raises(ValueError, match="CUDA"):
                    sq(A, W, *scales, o, activation=act, out_dtype=dt)
    # out_scale of scale_c's shape in both layouts reaches the CUDA check; other shapes, dtypes and layouts do not
    for good in (torch.ones(T, nb), torch.ones(nb, T).t()):
        with pytest.raises(ValueError, match="CUDA"):
            sq(x, W, *row_grp, offs, out_scale=good)
    for good in (torch.ones(G, m, nb), torch.ones(G, nb, m).transpose(1, 2)):
        with pytest.raises(ValueError, match="CUDA"):
            sq(x3, W, *row_bat, out_scale=good)
    for bad in (torch.ones(T, nb + 1), torch.ones(T, nb, dtype=torch.float64), torch.ones(G, T, nb),
                torch.ones(T * nb).as_strided((T, nb), (2, 1))):
        with pytest.raises(ValueError, match="out_scale"):
            sq(x, W, *row_grp, offs, out_scale=bad)
    with pytest.raises(ValueError, match="overlap"):                    # 3-D entries that overlap
        sq(x3, W, *row_bat, out_scale=torch.ones(G * m * nb).as_strided((G, m, nb), (m * nb - 1, nb, 1)))
    # the parent's refusals, and this call's own
    with pytest.raises(ValueError, match="out_dtype"):
        sq(x, W, *row_grp, offs, out_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="activation"):
        sq(x, W, *row_grp, offs, activation="tanh")
    with pytest.raises(ValueError, match="use_fast_accum"):
        sq(x, W, *blk_grp[0], offs, use_fast_accum=True)
    with pytest.raises(ValueError, match="offs"):
        sq(x, W, *row_grp)
    with pytest.raises(ValueError, match="out must"):
        sq(x, W, *row_grp, offs, out_dtype=torch.float8_e4m3fn, out=torch.empty(T, n, dtype=torch.float8_e5m2))
    with pytest.raises(ValueError, match="out must"):
        sq(x, W, *row_grp, offs, out_dtype=torch.float8_e4m3fn, out=torch.empty(T, n + 1, dtype=torch.float8_e4m3fn))
    with pytest.raises(TypeError):
        sq(_fp8((T, k), E5M2), _fp8((G, n, k), E5M2).transpose(-2, -1), *row_grp, offs)
    with pytest.raises(ValueError, match="B must be 3-D"):
        sq(x, _fp8((k, n)), *row_grp, offs)
    # scaled_grouped_mm keeps refusing an FP8 out_dtype
    for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
        with pytest.raises(ValueError, match="out_dtype"):
            gemm.scaled_grouped_mm(x, W, *row_grp, offs, out_dtype=dt)


# ==== GPU: problems with poisoned padding =========================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


class Out:
    """An FP8 C of `entries` x rows x n at pitch ldc (an odd pitch and an odd base by default) with `gap` bytes between
    entries, and its scales (row-major or outer-dim-major per entry, `sc_gap` floats between entries), all inside
    fence-filled buffers."""

    def __init__(self, entries, rows, n, ldc=None, base=1, gap=0, sc_layout="row", sc_gap=0):
        self.entries, self.rows, self.n = entries, rows, n
        self.ldc = n + 3 if ldc is None else ldc
        self.base, self.stride_c = base, rows * self.ldc + gap
        self.C = torch.full((base + entries * self.stride_c + 16,), C_FENCE, dtype=torch.uint8, device="cuda")
        self.qn = cdiv(n, 128)
        self.sc_layout = sc_layout
        self.sc_row, self.sc_blk = (self.qn, 1) if sc_layout == "row" else (1, rows)
        self.sc_e = rows * self.qn + sc_gap
        self.S = torch.full((8 + entries * self.sc_e + 8,), SC_SENTINEL, dtype=torch.int32, device="cuda")

    def c_ptr(self, e=0):
        return self.C.data_ptr() + self.base + e * self.stride_c

    def s_ptr(self, e=0):
        return self.S.data_ptr() + 4 * (8 + e * self.sc_e)

    def bytes(self):
        """(C bytes, scale bits) as numpy copies."""
        torch.cuda.synchronize()
        return self.C.cpu().numpy(), self.S.cpu().numpy()

    def entry(self, cb, sb, e, rows=None):
        """Entry e's (C, d): rows x n bytes and rows x q_n float32 scales."""
        rows = self.rows if rows is None else rows
        o = self.base + e * self.stride_c
        c = cb[o:o + rows * self.ldc].reshape(rows, self.ldc)[:, :self.n] if rows else np.zeros((0, self.n), np.uint8)
        s = sb[8 + e * self.sc_e:8 + e * self.sc_e + self.rows * self.qn].view(np.float32)
        d = s.reshape(self.rows, self.qn) if self.sc_layout == "row" else s.reshape(self.qn, self.rows).T
        return np.ascontiguousarray(c), np.ascontiguousarray(d[:rows])


def same_out(got, want, ct):
    """Two Out buffers hold the same bytes: C equal byte for byte, or NaN at the same places (NaN has two FP8 codes);
    scale_c equal bit for bit, or NaN at the same places."""
    (gc, gs), (wc, ws) = got.bytes(), want.bytes()
    gf, wf = gs.view(np.float32), ws.view(np.float32)
    return fo.same_fp8(gc, wc, ct) and fo.same_f32(gf, wf)


class Stacked:
    """A grouped (sizes or offs) or batched problem with a rowwise or blockwise input recipe; operands at padded
    pitches with FP8-NaN padding, scales NaN-padded between rows, k-blocks and entries."""

    def __init__(self, recipe, ta, tb, n, k, seed, sizes=None, offs=None, total_m=None, batch=None, m=None,
                 exact=False, broadcast_a=False):
        self.recipe, self.ta, self.tb, self.n, self.k = recipe, ta, tb, n, k
        self.grouped = batch is None
        rng = np.random.default_rng(seed)
        if self.grouped:
            self.G = len(sizes) if offs is None else len(offs)
            self.offs_list = list(np.cumsum(sizes)) if offs is None else list(offs)
            self.total_m = total_m if total_m is not None else int(sum(sizes))
            self.ends = gg.clamped_ends(self.offs_list, self.total_m)
            self.rows = self.total_m
            self.a8, self.b8, sa, sb = fg.operands(rng, ta, tb, self.total_m, n, k, self.G, exact)
            self.A, self.lda, _ = fg.padded(self.a8, pad16(k) + 16)
            self.stride_a = 0
            self.offs = torch.tensor([int(o) for o in self.offs_list], dtype=torch.int32, device="cuda")
        else:
            self.G, self.m, self.rows = batch, m, m
            a8, self.b8, sa, sb = fg.operands(rng, ta, tb, m, n, k, batch, exact)
            self.a8 = np.broadcast_to(a8, (batch, m, k)) if broadcast_a else \
                fg.operands(rng, ta, tb, batch * m, 1, k, 1, exact)[0].reshape(batch, m, k)
            self.A, self.lda, self.stride_a = fg.padded(a8 if broadcast_a else self.a8, pad16(k) + 16, entry_gap=32)
            if broadcast_a:
                self.stride_a = 0
            sa = fg.operands(rng, ta, tb, batch * m, 1, 1, 1, exact)[2].reshape(batch, m)
        self.B, self.ldb, self.stride_b = fg.padded(self.b8, pad16(k) + 32, entry_gap=48)
        if recipe[0] == "row":
            self.sa, self.sb = sa, sb                                           # (rows,) or (G, m); (G, n)
            self.Sa = bg.nan_padded(self.sa.reshape(1, -1))[0] if self.grouped else bg.nan_padded(self.sa)
            self.Sb = bg.nan_padded(self.sb)
        else:
            a_blk, b_blk = recipe[1]
            q = cdiv(k, 128)
            cols = cdiv(n, 128) if b_blk == 128 else n
            if self.grouped:
                self.sa = bg.make_scales(rng, (self.total_m, q), exact)
            else:
                self.sa = bg.make_scales(rng, (batch, m if a_blk == 1 else cdiv(m, 128), q), exact)
            self.sb = bg.make_scales(rng, (self.G, q, cols), exact)
            self.Sa, self.Sb = bg.nan_padded(self.sa), bg.nan_padded(self.sb)

    def fast(self, hooks):
        mode = self.recipe[1] if self.recipe[0] == "row" else "acc"
        return fg.set_mode(hooks, mode)

    def out(self, **kw):
        return Out(1 if self.grouped else self.G, self.rows, self.n, **kw)

    def call(self, gemm, hooks, o, ct, act, k=None, stream=None):
        """The stacked _q8 call into Out o."""
        fast = self.fast(hooks)
        k = self.k if k is None else k
        ssb = self.Sb.stride(0) if self.G > 1 else 0
        lib = gemm.lib
        if self.recipe[0] == "row" and self.grouped:
            rc = lib.b200_gemm_fp8_grouped_q8(self.ta, self.tb, self.total_m, self.n, k, self.A.data_ptr(), self.lda,
                                              self.B.data_ptr(), self.ldb, self.stride_b, self.offs.data_ptr(), self.G,
                                              self.Sa.data_ptr(), self.Sb.data_ptr(), ssb, act, fast, ct, o.c_ptr(),
                                              o.ldc, o.s_ptr(), o.sc_row, o.sc_blk, stream)
        elif self.recipe[0] == "row":
            rc = lib.b200_gemm_fp8_batched_q8(self.ta, self.tb, self.m, self.n, k, self.A.data_ptr(), self.lda,
                                              self.stride_a, self.B.data_ptr(), self.ldb, self.stride_b, self.Sa.data_ptr(),
                                              self.Sa.stride(0), self.Sb.data_ptr(), ssb, act, fast, ct, o.c_ptr(), o.ldc,
                                              o.stride_c, o.s_ptr(), o.sc_row, o.sc_blk, o.sc_e, self.G, stream)
        elif self.grouped:
            Sa, Sb = self.Sa, self.Sb
            rc = lib.b200_gemm_fp8_blockwise_grouped_q8(
                self.ta, self.tb, self.total_m, self.n, k, self.A.data_ptr(), self.lda, self.B.data_ptr(), self.ldb,
                self.stride_b, self.offs.data_ptr(), self.G, Sa.data_ptr(), Sa.stride(0), Sa.stride(1), Sb.data_ptr(),
                self.recipe[1][1], Sb.stride(1), Sb.stride(2), ssb, act, ct, o.c_ptr(), o.ldc, o.s_ptr(), o.sc_row,
                o.sc_blk, stream)
        else:
            Sa, Sb = self.Sa, self.Sb
            rc = lib.b200_gemm_fp8_blockwise_batched_q8(
                self.ta, self.tb, self.m, self.n, k, self.A.data_ptr(), self.lda, self.stride_a, self.B.data_ptr(),
                self.ldb, self.stride_b, Sa.data_ptr(), self.recipe[1][0], Sa.stride(1), Sa.stride(2),
                Sa.stride(0) if self.G > 1 else 0, Sb.data_ptr(), self.recipe[1][1], Sb.stride(1), Sb.stride(2), ssb,
                act, ct, o.c_ptr(), o.ldc, o.stride_c, o.s_ptr(), o.sc_row, o.sc_blk, o.sc_e, self.G, stream)
        assert rc == 0, rc
        return rc

    def entries(self):
        """(entry, first row of its C / scales in the Out, rows, A rows) of every entry with rows."""
        if self.grouped:
            lo = 0
            for g, hi in enumerate(self.ends):
                if hi > lo:
                    yield g, lo, hi - lo, self.a8[lo:hi], (self.sa[lo:hi] if self.recipe[0] == "row" else self.sa[lo:hi])
                lo = hi
        else:
            for e in range(self.G):
                yield e, None, self.m, np.ascontiguousarray(self.a8[e]), self.sa[e]

    def reference(self, gemm, hooks, like, ct, act, k=None):
        """Each entry by the single-matrix _q8 / _blockwise_q8 call (N, T), dynamic mode, null bias, on contiguous
        aligned copies of its rows, B and scales, into an Out shaped like `like`."""
        o = Out(like.entries, like.rows, like.n, ldc=like.ldc, base=like.base, gap=like.stride_c - like.rows * like.ldc,
                sc_layout=like.sc_layout, sc_gap=like.sc_e - like.rows * like.qn)
        fast = self.fast(hooks)
        k = self.k if k is None else k
        for e, lo, rows, a8, sa in self.entries():
            A, lda, _ = fg.padded(a8, pad16(self.k))
            B, ldb, _ = fg.padded(self.b8[e], pad16(self.k))
            if lo is None:
                cp, sp = o.c_ptr(e), o.s_ptr(e)
            else:
                cp = o.c_ptr() + lo * o.ldc
                sp = o.s_ptr() + 4 * lo * o.sc_row
            if self.recipe[0] == "row":
                Sa, Sb = dev(sa), dev(self.sb[e])
                rc = gemm.lib.b200_gemm_fp8_q8(OP_N, OP_T, self.ta, self.tb, rows, self.n, k, A.data_ptr(), lda,
                                               B.data_ptr(), ldb, Sa.data_ptr(), 1, Sb.data_ptr(), 1, None, act, fast, ct,
                                               cp, o.ldc, None, sp, o.sc_row, o.sc_blk, None)
            else:
                Sa, Sb = dev(sa), dev(self.sb[e])
                rc = gemm.lib.b200_gemm_fp8_blockwise_q8(
                    OP_N, OP_T, self.ta, self.tb, rows, self.n, k, A.data_ptr(), lda, B.data_ptr(), ldb, Sa.data_ptr(),
                    self.recipe[1][0] if not self.grouped else 1, *bw.strides_of(Sa), Sb.data_ptr(), self.recipe[1][1],
                    *bw.strides_of(Sb), None, act, ct, cp, o.ldc, None, sp, o.sc_row, o.sc_blk, None)
            assert rc == 0, rc
        torch.cuda.synchronize()
        return o

    def check(self, gemm, hooks, ct, act, stack, out_kw=None, k=None):
        """The stacked call equals the per-entry reference over both whole buffers, fences included."""
        o = self.out(**(out_kw or {}))
        self.call(gemm, hooks, o, ct, act, k=k)
        torch.cuda.synchronize()
        kernel = gemm.last_kernel()
        want = self.reference(gemm, hooks, o, ct, act, k=k)
        assert same_out(o, want, ct), (self.recipe, ct, act, stack)
        return o, kernel


def check_fences(P, o):
    """Nothing written past each entry's rows (a grouped call's rows from end_{G-1} on), n, ldc, or the scales'."""
    cb, sb = o.bytes()
    assert (cb[:o.base] == C_FENCE).all() and (cb[o.base + o.entries * o.stride_c:] == C_FENCE).all()
    for e in range(o.entries):
        body = cb[o.base + e * o.stride_c:o.base + e * o.stride_c + o.rows * o.ldc].reshape(o.rows, o.ldc)
        assert (body[:, P.n:] == C_FENCE).all()
        assert (cb[o.base + e * o.stride_c + o.rows * o.ldc:o.base + (e + 1) * o.stride_c] == C_FENCE).all()
        last = P.ends[-1] if P.grouped else o.rows
        assert (body[last:] == C_FENCE).all()
        s = sb[8 + e * o.sc_e:8 + e * o.sc_e + o.rows * o.qn]
        d = s.reshape(o.rows, o.qn) if o.sc_layout == "row" else s.reshape(o.qn, o.rows).T
        assert (d[last:] == SC_SENTINEL).all() and not (d[:last] == SC_SENTINEL).any()
        assert (sb[8 + e * o.sc_e + o.rows * o.qn:8 + (e + 1) * o.sc_e] == SC_SENTINEL).all()
    assert (sb[:8] == SC_SENTINEL).all() and (sb[8 + o.entries * o.sc_e:] == SC_SENTINEL).all()


# the grouped offsets: empty groups, 1-row groups, a decreasing offset, the last past total_m (clamped), rows after
# the last group that stay untouched
OFFS = ([0, 1, 129, 129, 300, 420, 380, 1000], 700)
OFFS_TAIL = ([127, 127, 427, 428, 300, 556], 700)


@gpu
@pytest.mark.parametrize("ct", [E4M3, E5M2], ids=lambda c: CT_NAME[c])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_bit_identical_to_single_matrix_per_entry(gemm, hooks, pair, ct):
    """Every recipe of the case table, every activation: each group / entry equals the single-matrix _q8 call on
    its own rows, B and scales (whole buffers, fences and untouched rows included); last_kernel() names the case's
    kernel.  n = 300 (a tail block), k = 416 (a k tail), odd ldc and an odd C base."""
    seed = 3 * PAIRS.index(pair) + ct
    for _, _, stack, recipe in [c for c in case_table() if c[0] == pair and c[1] == ct]:
        if stack == "grp":
            offs, total_m = OFFS if recipe[1] != (1, 1) else OFFS_TAIL
            P = Stacked(recipe, *pair, 300, 416, seed, offs=offs, total_m=total_m)
        else:
            P = Stacked(recipe, *pair, 300, 416, seed, batch=3, m=150, broadcast_a=recipe[0] == "blk")
        for act in ACTS:
            o, kernel = P.check(gemm, hooks, ct, act, stack, out_kw={"sc_layout": "outer" if act % 2 else "row",
                                                                     "gap": 5, "sc_gap": 3})
            assert kernel == kernel_name(*pair, ct, stack, recipe), (kernel, recipe)
            check_fences(P, o)


@gpu
@pytest.mark.parametrize("stack", ["grp", "bat"])
def test_exact_oracle(gemm, hooks, stack):
    """Integer operands and power-of-two scales: each entry is quant_dynamic of the exact fp32 oracle, bit for bit, for
    the promoted, a fast and a blockwise recipe, with ReLU."""
    for recipe in (("row", "acc"), ("row", 128), ("blk", (1, 128))):
        for ct in (E4M3, E5M2):
            if stack == "grp":
                P = Stacked(recipe, E4M3, E4M3, 200, 384, 5, sizes=[130, 0, 1, 257, 40], exact=True)
            else:
                P = Stacked(recipe, E4M3, E4M3, 200, 384, 5, batch=2, m=130, exact=True)
            o = P.out()
            P.call(gemm, hooks, o, ct, fo.ACT_RELU)
            cb, sb = o.bytes()
            for e, lo, rows, a8, sa in P.entries():
                a = f8.decode(a8, E4M3)
                b = f8.decode(P.b8[e], E4M3).T
                if recipe[0] == "row":
                    v = f8.oracle(a, b, sa, P.sb[e], None, f8.OUT_F32)
                else:
                    sa_full, sb_full = bw.expand_scales(sa, P.sb[e], recipe[1], rows, P.n)
                    v = bw.oracle_blockwise(a, b, sa_full, sb_full, None, f8.OUT_F32)
                wq, wd = fo.quant_dynamic(fo.relu_np(v.astype(np.float32)), ct)
                if lo is None:
                    c, d = o.entry(cb, sb, e)
                else:
                    c, d = o.entry(cb, sb, 0)
                    c, d = c[lo:lo + rows], d[lo:lo + rows]
                assert fo.same_fp8(c, wq, ct) and fo.same_f32(d, wd), (recipe, ct, e)


@gpu
@pytest.mark.parametrize("recipe", [("row", "acc"), ("row", 256), ("row", 128), ("blk", (1, 128))], ids=RECIPE_ID)
def test_schedules(gemm, hooks, sms, recipe):
    """Two full rounds of tiles over the SMs plus a partial one, 7 k-blocks (more than any width's stages), a group of
    17 tile rows and forced raster group rows that make the last raster group ragged: grouped and batched."""
    n, k = 640, 7 * 128 - 16
    try:
        for rows in (0, 384):
            gemm.lib.b200_gemm_debug_set_group_rows(rows)
            P = Stacked(recipe, E4M3, E4M3, n, k, 9, sizes=[2176, 3000, 1, 0, 4100, 2900])
            width = 128 if recipe[1] in ("acc", 128) or recipe[0] == "blk" else 256
            tiles = sum(cdiv(s, 128) for s in (2176, 3000, 1, 4100, 2900)) * cdiv(n, width)
            assert tiles > 2 * sms and tiles % sms, tiles
            P.check(gemm, hooks, E4M3, fo.ACT_GELU, "grp")
            P = Stacked(recipe, E4M3, E5M2, n, k, 10, batch=6, m=2176)
            assert 6 * 17 * cdiv(n, width) > 2 * sms
            P.check(gemm, hooks, E5M2, fo.ACT_NONE, "bat")
    finally:
        gemm.lib.b200_gemm_debug_set_group_rows(0)


@gpu
def test_many_groups_and_narrow_outputs(gemm, hooks):
    """256 Zipf-sized groups; n below 128 and n = 129 (a one-column tail block), odd ldc, odd C base."""
    rng = np.random.default_rng(7)
    sizes = list((1000 / np.arange(1, 257) ** 1.1).astype(int))
    for recipe in (("row", 128), ("blk", (1, 1))):
        P = Stacked(recipe, E4M3, E4M3, 256, 128, 11, sizes=sizes)
        P.check(gemm, hooks, E4M3, fo.ACT_RELU, "grp")
    for n in (100, 129):
        for recipe in (("row", "acc"), ("row", 256), ("blk", (128, 1))):
            P = Stacked(recipe, E5M2, E4M3, n, 200, int(rng.integers(99)), batch=3, m=70)
            o, _ = P.check(gemm, hooks, E4M3, fo.ACT_NONE, "bat", out_kw={"ldc": n + 1, "base": 3})
            check_fences(P, o)


@gpu
def test_non_finite_blocks_and_saturation(gemm, hooks):
    """NaN operand bytes and an inf scale make their rows' blocks NaN with d = NaN; large values saturate to +-F.
    Equal to the single-matrix reference bit for bit (NaN at the same places)."""
    for recipe in (("row", "acc"), ("row", 256), ("blk", (1, 128))):
        P = Stacked(recipe, E4M3, E4M3, 300, 256, 13, sizes=[100, 50, 150])
        a8 = P.a8.copy()
        a8[3, 5] = fg.NAN8
        a8[120, 7] = fg.NAN8
        P.a8 = a8
        P.A, P.lda, _ = fg.padded(a8, pad16(P.k) + 16)
        sa = P.sa.copy()
        if recipe[0] == "row":
            sa[60] = np.inf
            sa[61] = 1e30
        else:
            sa[60, 1] = np.inf
            sa[61, 0] = 1e30
        P.sa = sa
        P.Sa = bg.nan_padded(sa.reshape(1, -1))[0] if recipe[0] == "row" else bg.nan_padded(sa)
        for ct in (E4M3, E5M2):
            o, _ = P.check(gemm, hooks, ct, fo.ACT_NONE, "grp")
            cb, sb = o.bytes()
            c, d = o.entry(cb, sb, 0)
            assert np.isnan(d[3]).any() and np.isnan(d[120]).any() and np.isnan(d[60]).all()
            assert np.isfinite(d[61]).all() and (np.abs(f8.decode(c[61], ct)) <= float(fo.FMAX[ct])).all()


@gpu
def test_k_zero(gemm, hooks):
    """k == 0: act(+0) quantised (the +0 byte) and d = 1 over the covered rows / entries, nothing else written, no
    operand or scale read (null pointers); bit for bit the single-matrix k == 0 call."""
    for recipe in (("row", "acc"), ("blk", (1, 128))):
        for act in ACTS:
            P = Stacked(recipe, E4M3, E4M3, 300, 128, 17, offs=OFFS_TAIL[0], total_m=OFFS_TAIL[1])
            o, kernel = P.check(gemm, hooks, E4M3, act, "grp", k=0)
            assert kernel == "fp8_q8_k0_grp"
            check_fences(P, o)
            cb, sb = o.bytes()
            c, d = o.entry(cb, sb, 0, rows=P.ends[-1])
            assert (c == 0).all() and (d == 1).all()
            P = Stacked(recipe, E4M3, E4M3, 300, 128, 17, batch=3, m=50)
            o, kernel = P.check(gemm, hooks, E5M2, act, "bat", k=0)
            assert kernel == "fp8_q8_k0_bat"
            check_fences(P, o)


@gpu
def test_batch_of_one_is_the_single_matrix_call(gemm, hooks):
    for recipe, name in ((("row", "acc"), "tc_e4m3_oe4m3_acc_128x128"), (("row", 256), "tc_e4m3_oe4m3_128x256"),
                         (("blk", (128, 1)), "tc_e4m3_oe4m3_blk_128x128")):
        P = Stacked(recipe, E4M3, E4M3, 300, 256, 19, batch=1, m=200)
        o, kernel = P.check(gemm, hooks, E4M3, fo.ACT_GELU, "bat")
        assert kernel == name, kernel


@gpu
def test_cuda_graph_replay_with_new_offsets_and_scales(gemm, hooks):
    """Captured once; offsets and scales rewritten on the device between replays; each replay equals the reference."""
    for recipe in (("row", 128), ("blk", (1, 128))):
        P = Stacked(recipe, E4M3, E4M3, 256, 256, 23, sizes=[100, 200, 0, 300])
        o = P.out()
        s = torch.cuda.Stream()
        P.fast(hooks)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            P.call(gemm, hooks, o, E4M3, fo.ACT_RELU, stream=s.cuda_stream)
        for step, offs in enumerate(([100, 200, 0, 300], [250, 250, 400, 600], [0, 600, 10, 300])):
            P.offs.copy_(torch.tensor(offs, dtype=torch.int32))
            P.offs_list, P.ends = offs, gg.clamped_ends(offs, P.total_m)
            P.sa = (P.sa * np.float32(2.0 if step else 1.0)).astype(np.float32)
            P.Sa.copy_(dev(P.sa))
            o.C.fill_(C_FENCE)
            o.S.fill_(SC_SENTINEL)
            g.replay()
            torch.cuda.synchronize()
            want = P.reference(gemm, hooks, o, E4M3, fo.ACT_RELU)
            assert same_out(o, want, E4M3), (recipe, step)
            check_fences(P, o)


@gpu
def test_chain_into_the_next_grouped_gemm(gemm, hooks):
    """scaled_grouped_mm_quant -> scaled_grouped_mm (blockwise, 128 x 128 down-projection scales) equals the per-group
    single-matrix chain scaled_mm_quant -> scaled_mm bit for bit, for a 2-D and a 3-D A."""
    rng = np.random.default_rng(29)
    G, d, dff = 4, 256, 384
    sizes = [130, 0, 1, 300]
    T = sum(sizes)
    offs = torch.tensor(np.cumsum(sizes), dtype=torch.int32, device="cuda")
    x = dev(f8.encode(rng.standard_normal((T, d)), E4M3)).view(torch.float8_e4m3fn)
    W1 = dev(f8.encode(rng.standard_normal((G, dff, d)), E4M3)).view(torch.float8_e4m3fn)
    W2 = dev(f8.encode(rng.standard_normal((G, d, dff)), E4M3)).view(torch.float8_e4m3fn)
    q1, q2 = cdiv(d, 128), cdiv(dff, 128)
    sx, sw1 = dev(bw.random_scales(rng, (T, q1))), dev(bw.random_scales(rng, (G, q1, cdiv(dff, 128))))
    sw2 = dev(bw.random_scales(rng, (G, q2, cdiv(d, 128))))
    h, sh = gemm.scaled_grouped_mm_quant(x, W1.transpose(-2, -1), sx, sw1, offs, activation="gelu")
    assert h.dtype == torch.float8_e4m3fn and sh.shape == (T, q2)
    assert gemm.last_kernel() == "tc_e4m3_oe4m3_grp_blk_128x128"
    y = gemm.scaled_grouped_mm(h, W2.transpose(-2, -1), sh, sw2, offs, out_dtype=torch.float32)
    ends = [0] + offs.tolist()
    for g in range(G):
        lo, hi = ends[g], ends[g + 1]
        if hi == lo:
            continue
        hg, shg = gemm.scaled_mm_quant(x[lo:hi], W1[g].t(), sx[lo:hi], sw1[g], activation="gelu")
        assert torch.equal(h[lo:hi].view(torch.uint8), hg.view(torch.uint8)) and torch.equal(sh[lo:hi], shg)
        yg = gemm.scaled_mm(hg, W2[g].t(), shg, sw2[g], out_dtype=torch.float32)
        assert torch.equal(y[lo:hi], yg), g
    # a 3-D A, rowwise up projection with fast accumulation, both at the same forced width
    hooks.b200_gemm_debug_set_bn(128)
    m = 200
    x3 = dev(f8.encode(rng.standard_normal((G, m, d)), E4M3)).view(torch.float8_e4m3fn)
    sa3, sb3 = dev(bw.random_scales(rng, (G, m))), dev(bw.random_scales(rng, (G, dff)))
    h3, sh3 = gemm.scaled_grouped_mm_quant(x3, W1.transpose(-2, -1), sa3, sb3, use_fast_accum=True,
                                           out_dtype=torch.float8_e5m2, activation="relu")
    assert sh3.shape == (G, m, q2) and h3.dtype == torch.float8_e5m2
    y3 = gemm.scaled_grouped_mm(h3, W2.transpose(-2, -1), sh3, sw2, out_dtype=torch.float32)
    for g in range(G):
        hg, shg = gemm.scaled_mm_quant(x3[g], W1[g].t(), sa3[g][:, None], sb3[g][None, :], use_fast_accum=True,
                                       out_dtype=torch.float8_e5m2, activation="relu")
        assert torch.equal(h3[g].view(torch.uint8), hg.view(torch.uint8)) and torch.equal(sh3[g], shg)
        assert torch.equal(y3[g], gemm.scaled_mm(hg, W2[g].t(), shg, sw2[g], out_dtype=torch.float32)), g


@gpu
def test_deepseek_v3_sized_chain(gemm):
    """A DeepSeek-V3-sized expert FFN (d = 7168, d_ff = 2048, routed tokens over 8 experts): the fused up projection's
    (C, scale_c) feeds the blockwise down projection, each within the existing blockwise bound of the float64 product
    of its own quantised inputs."""
    torch.manual_seed(19)
    G, d, dff = 8, 7168, 2048
    sizes = [700, 40, 0, 513, 300, 1, 900, 94]
    offs = torch.tensor(np.cumsum(sizes), dtype=torch.int32, device="cuda")
    x = torch.randn((sum(sizes), d), device="cuda")
    W1 = torch.randn((G, dff, d), device="cuda") * 0.02
    W2 = torch.randn((G, d, dff), device="cuda") * 0.02
    xq, sx = bg.quantise_1x128(x)
    w1q, sw1 = bg.quantise_128x128(W1)
    w2q, sw2 = bg.quantise_128x128(W2)
    h, sh = gemm.scaled_grouped_mm_quant(xq, w1q.transpose(-2, -1), sx.t().contiguous().t(), sw1.transpose(1, 2), offs,
                                         activation="relu")
    assert gemm.last_kernel() == "tc_e4m3_oe4m3_grp_blk_128x128"
    y = gemm.scaled_grouped_mm(h, w2q.transpose(-2, -1), sh, sw2.transpose(1, 2), offs, out_dtype=torch.float32)
    ends = [0] + offs.tolist()
    for g in range(G):
        lo, hi = ends[g], ends[g + 1]
        if hi == lo:
            continue
        rows = torch.arange(lo, hi, 37, device="cuda")
        # layer 1: the dequantised h within the fp32 bound plus one e4m3 rounding (2^-4 relative, or half the
        # smallest subnormal 2^-10 times the block scale)
        a, b = xq[rows].float().cpu().numpy(), w1q[g].float().cpu().numpy().T
        ex, w = bw.exact_and_weight(a, b, sx[rows].cpu().numpy(), np.repeat(sw1[g].t().cpu().numpy(), 128, axis=1))
        ex = np.maximum(ex, 0)
        dq = np.repeat(sh[rows].cpu().numpy().astype(np.float64), 128, axis=1)
        hd = h[rows].float().cpu().numpy().astype(np.float64) * dq
        quant = 2.0 ** -4 * np.abs(ex) + 2.0 ** -10 * dq
        assert bool((np.abs(hd - ex) <= 1.07 * bw.rel_bound(d) * w + quant).all()), g
        # layer 2: on its own quantised inputs, the blockwise bound
        a2, b2 = h[rows].float().cpu().numpy(), w2q[g].float().cpu().numpy().T
        ex2, w2 = bw.exact_and_weight(a2, b2, sh[rows].cpu().numpy(), np.repeat(sw2[g].t().cpu().numpy(), 128, axis=1))
        assert bool((np.abs(y[rows].double().cpu().numpy() - ex2) <= bw.rel_bound(dff) * w2).all()), g
