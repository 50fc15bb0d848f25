"""Grouped and batched FP8 GEMMs (b200_gemm_fp8_grouped / _batched) and scaled_grouped_mm(): torch._scaled_grouped_mm's
2-D x 3-D and 3-D x 3-D forms for FP8 mixture-of-experts layers.

Every group (rows [end_{g-1}, end_g) of A and C, times B_g) and every batch entry is one (N, T) b200_gemm_fp8 call with
rowwise scales: C = round_out((acc * sa_i) * sb_j).  The stacked kernels run the same MMA chains and epilogue, so with
the tile width forced each group must equal b200_gemm_fp8 on contiguous copies of its rows of A and scale_a, of B_g and
of row g of scale_b, bit for bit.  Output buffers start as NaN and the operands' padding holds FP8 NaN bytes, and whole
buffers are compared, so a row written to the wrong place, a row past the last group written, or a padding byte read
cannot pass.  On integer operands with power-of-two scales acc is exact, and the results must equal a numpy model of
rn(rn(acc * sa) * sb) rounded to the output type.

The argument checks and the Python refusals need no GPU."""
import math

import numpy as np
import pytest

import test_batched_gpu as bt
import test_fp8_gpu as f8
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
OUTS = (OUT_F32, OUT_BF16, OUT_F16)
MODES = ("acc", 256, 192, 128)          # promoted (128 x 128), or fast at a forced width
NAN8 = 0x7F                             # NaN in both e4m3 and e5m2
ERR_BAD_ARG, ERR_NO_DEVICE, ERR_UNSUPPORTED = -1, -2, -3
_has_gpu = f8._has_gpu


def pad16(x):
    return (x + 15) // 16 * 16


def kernel_name(ta, tb, o, stack, mode):
    width = "acc_128x128" if mode == "acc" else f"128x{mode}"
    return f"tc_{PAIR_NAME[(ta, tb)]}_{OUT_NAME[o]}_{stack}_{width}"


# ==== the C ABI through ctypes (CPU: every refusal happens before the device is touched) =============================
def call_grp(gemm, ta=E4M3, tb=E4M3, total_m=40, n=32, k=32, a=16, lda=None, b=16, ldb=None, stride_b=None, offs=16,
             groups=3, sa=16, sb=16, ssb=32, c=16, ldc=None, out=OUT_BF16, fast=0):
    """b200_gemm_fp8_grouped with raw pointers (16 stands for a dummy aligned non-null pointer, 1 for a misaligned one)."""
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    return gemm.lib.b200_gemm_fp8_grouped(ta, tb, total_m, n, k, a, lda, b, ldb, stride_b, offs, groups, sa, sb, ssb, c,
                                          ldc, out, fast, None)


def call_bat(gemm, ta=E4M3, tb=E4M3, m=40, n=32, k=32, a=16, lda=None, stride_a=None, b=16, ldb=None, stride_b=None,
             sa=16, ssa=40, sb=16, ssb=32, c=16, ldc=None, stride_c=None, batch=3, out=OUT_BF16, fast=0):
    lda = k if lda is None else lda
    ldb = k if ldb is None else ldb
    stride_a = m * lda if stride_a is None else stride_a
    stride_b = n * ldb if stride_b is None else stride_b
    ldc = n if ldc is None else ldc
    stride_c = m * ldc if stride_c is None else stride_c
    return gemm.lib.b200_gemm_fp8_batched(ta, tb, m, n, k, a, lda, stride_a, b, ldb, stride_b, sa, ssa, sb, ssb, c, ldc,
                                          stride_c, batch, out, fast, None)


def test_grouped_argument_validation(gemm):
    """Refusals before the device is touched, each at its bound: they hold with or without a GPU."""
    for call in (call_grp, call_bat):
        assert call(gemm, ta=2) == ERR_BAD_ARG and call(gemm, tb=-1) == ERR_BAD_ARG
        assert call(gemm, out=3) == ERR_BAD_ARG and call(gemm, out=-1) == ERR_BAD_ARG
        assert call(gemm, fast=2) == ERR_BAD_ARG and call(gemm, fast=-1) == ERR_BAD_ARG
        assert call(gemm, n=-1) == ERR_BAD_ARG and call(gemm, k=-1) == ERR_BAD_ARG
        assert call(gemm, ta=E5M2, tb=E5M2) == ERR_UNSUPPORTED                     # as b200_gemm_fp8
        assert call(gemm, ldb=31) == ERR_BAD_ARG                                    # B_g is n x k: ldb >= k
        assert call(gemm, lda=31) == ERR_BAD_ARG and call(gemm, ldc=31) == ERR_BAD_ARG
        assert call(gemm, a=None) == ERR_BAD_ARG and call(gemm, b=None) == ERR_BAD_ARG
        assert call(gemm, c=None) == ERR_BAD_ARG
        assert call(gemm, sa=None) == ERR_BAD_ARG and call(gemm, sb=None) == ERR_BAD_ARG
        assert call(gemm, sa=None, k=0, a=None, b=None) == ERR_BAD_ARG              # a null scale with work to do
        assert call(gemm, ssb=-1) == ERR_BAD_ARG
        assert call(gemm, n=0, a=None, b=None, c=None, sa=None, sb=None) == 0      # no-ops
        # operands the tensor cores cannot read in place
        assert call(gemm, a=1) == ERR_UNSUPPORTED and call(gemm, b=1 + 16) == ERR_UNSUPPORTED
        assert call(gemm, k=24) == ERR_UNSUPPORTED                                  # lda = ldb = 24 bytes
        assert call(gemm, lda=40) == ERR_UNSUPPORTED and call(gemm, ldb=40) == ERR_UNSUPPORTED
    # grouped: b200_gemm_bf16_grouped's rules
    assert call_grp(gemm, total_m=-1) == ERR_BAD_ARG
    assert call_grp(gemm, groups=-1) == ERR_BAD_ARG and call_grp(gemm, groups=1025) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=-1) == ERR_BAD_ARG
    assert call_grp(gemm, offs=None) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=32 * 32 - 16) == ERR_BAD_ARG                     # B_g overlap
    assert call_grp(gemm, stride_b=0) == ERR_BAD_ARG                                # broadcast B is a torch refusal too
    assert call_grp(gemm, stride_b=(1 << 60) // 2 + 16) == ERR_BAD_ARG             # (groups - 1) * stride_b > 2^60
    assert call_grp(gemm, ssb=(1 << 60) // 2 + 1) == ERR_BAD_ARG
    assert call_grp(gemm, stride_b=32 * 32 + 8) == ERR_UNSUPPORTED                  # not a 16-byte multiple
    assert call_grp(gemm, stride_b=1 << 41) == ERR_UNSUPPORTED                      # beyond what TMA encodes
    assert call_grp(gemm, total_m=1 << 30, n=1 << 20) == ERR_BAD_ARG                # the tile bound
    assert call_grp(gemm, groups=0, a=None, b=None, c=None, offs=None, sa=None, sb=None) == 0
    assert call_grp(gemm, total_m=0, a=None, b=None, c=None, offs=None, sa=None, sb=None) == 0
    # batched: b200_gemm_bf16_batched's rules
    assert call_bat(gemm, m=-1) == ERR_BAD_ARG and call_bat(gemm, batch=-1) == ERR_BAD_ARG
    for kw in ("stride_a", "stride_b", "stride_c", "ssa", "ssb"):
        assert call_bat(gemm, **{kw: -1}) == ERR_BAD_ARG, kw
        assert call_bat(gemm, **{kw: (1 << 60) // 2 + 16}) == ERR_BAD_ARG, kw
    assert call_bat(gemm, stride_c=39 * 32 + 31) == ERR_BAD_ARG                     # entries of C overlap
    assert call_bat(gemm, m=1 << 21, n=1 << 21, batch=3) == ERR_BAD_ARG             # the tile bound
    assert call_bat(gemm, stride_a=40 * 32 - 16) == ERR_UNSUPPORTED                 # overlapping inputs
    assert call_bat(gemm, stride_b=32 * 32 - 16) == ERR_UNSUPPORTED
    assert call_bat(gemm, stride_a=40 * 32 + 8) == ERR_UNSUPPORTED
    assert call_bat(gemm, batch=0, a=None, b=None, c=None, sa=None, sb=None) == 0
    assert call_bat(gemm, m=0, a=None, b=None, c=None, sa=None, sb=None) == 0


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_grouped_accepts_at_the_bounds_without_device(gemm):
    """Legal calls at the bounds reach the device check (-2): broadcast A and B with their own scale strides, scale
    strides of 0, one group, k == 0 with null operands, every pair, C type and mode."""
    assert call_grp(gemm, groups=1, stride_b=0, ssb=0) == ERR_NO_DEVICE
    assert call_grp(gemm, groups=1024) == ERR_NO_DEVICE
    assert call_grp(gemm, stride_b=32 * 32, ssb=0) == ERR_NO_DEVICE
    assert call_grp(gemm, k=0, a=None, b=None) == ERR_NO_DEVICE
    assert call_grp(gemm, k=0, a=1, b=1) == ERR_NO_DEVICE                          # k == 0 reads no operand
    assert call_bat(gemm, k=0, a=1, b=1) == ERR_NO_DEVICE
    assert call_bat(gemm, stride_a=0, stride_b=0, ssa=7, ssb=0) == ERR_NO_DEVICE
    assert call_bat(gemm, batch=1, stride_a=-0, stride_c=0) == ERR_NO_DEVICE
    assert call_bat(gemm, k=0, a=None, b=None) == ERR_NO_DEVICE
    for ta, tb in PAIRS:
        for o in OUTS:
            for fast in (0, 1):
                assert call_grp(gemm, ta=ta, tb=tb, out=o, fast=fast) == ERR_NO_DEVICE
                assert call_bat(gemm, ta=ta, tb=tb, out=o, fast=fast) == ERR_NO_DEVICE


# ==== scaled_grouped_mm: refusals (CPU) ===========================================================================
def _fp8(shape, t=E4M3):
    return torch.zeros(shape, dtype=torch.float32).to(f8.fp8_dtype(t))


@need_torch
def test_scaled_grouped_mm_refusals(gemm):
    G, T, m, n, k = 3, 40, 8, 32, 64
    x, W = _fp8((T, k)), _fp8((G, n, k))
    B = W.transpose(-2, -1)                                  # (G, k, n), column-major: torch's mat_b
    xa = _fp8((G, m, k))
    offs = torch.tensor([10, 20, 40], dtype=torch.int32)
    sa, sb, sa3 = torch.ones(T), torch.ones(G, n), torch.ones(G, m)
    sgm = gemm.scaled_grouped_mm
    with pytest.raises(TypeError):
        sgm(x.float(), B, sa, sb, offs)
    with pytest.raises(TypeError):
        sgm(_fp8((T, k), E5M2), _fp8((G, n, k), E5M2).transpose(-2, -1), sa, sb, offs)
    with pytest.raises(ValueError, match="not supported"):
        sgm(x, _fp8((n, k)).t(), sa, torch.ones(n), offs)                   # 2-D x 2-D
    with pytest.raises(ValueError, match="not supported"):
        sgm(xa, _fp8((n, k)).t(), sa3, torch.ones(n))                       # 3-D x 2-D
    with pytest.raises(ValueError):
        sgm(x, B.contiguous(), sa, sb, offs)                                # B row-major in its last two dims
    with pytest.raises(ValueError):
        sgm(x.t().contiguous().t(), B, sa, sb, offs)                        # A column-major
    with pytest.raises(ValueError):
        sgm(x, _fp8((G, n, k + 16)).transpose(-2, -1), sa, sb, offs)        # contraction dims differ
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb)                                                   # 2-D A needs offs
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs.long())
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs[:2])
    with pytest.raises(ValueError):
        sgm(xa, B, sa3, sb, offs)                                           # 3-D A takes no offs
    with pytest.raises(ValueError):
        sgm(_fp8((G + 1, m, k)), B, torch.ones(G + 1, m), sb)
    with pytest.raises(ValueError):
        sgm(x, B, sa.double(), sb, offs)
    with pytest.raises(ValueError):
        sgm(x, B, torch.ones(T, 1), sb, offs)                               # scale_a (total_m,)
    with pytest.raises(ValueError):
        sgm(x, B, sa, torch.ones(G * n), offs)                              # scale_b (G, n)
    with pytest.raises(ValueError):
        sgm(x, B, sa, torch.ones(n, G).t(), offs)                           # scale_b contiguous along n
    with pytest.raises(ValueError):
        sgm(xa, B, torch.ones(G, m + 1), sb)
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs, out_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs, out_dtype=torch.bfloat16, out=torch.empty(T, n, dtype=torch.float16))
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs, out=torch.empty(T, n + 1, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        sgm(xa, B, sa3, sb, out=torch.empty(m * n, dtype=torch.bfloat16).as_strided((G, m, n), (0, n, 1)))
    with pytest.raises(ValueError):
        sgm(x, W[:1].expand(G, n, k).transpose(-2, -1), sa, sb, offs)      # broadcast B of a grouped call
    with pytest.raises(ValueError):
        sgm(x, B, sa, sb, offs)                                             # CPU tensors


# ==== GPU: problems with poisoned padding =========================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def operands(rng, ta, tb, rows, n, k, groups, exact):
    """FP8 bytes of A (rows x k) and of the groups' B_g^T (groups x n x k), and float32 rowwise scales: integer operands
    in [-2, 2] with power-of-two scales (exact = True), or random values with random scales."""
    if exact:
        a = rng.integers(-2, 3, (rows, k)).astype(np.float32)
        b = rng.integers(-2, 3, (groups, n, k)).astype(np.float32)
        sa = np.exp2(rng.integers(-3, 4, rows)).astype(np.float32)
        sb = np.exp2(rng.integers(-3, 4, (groups, n))).astype(np.float32)
    else:
        a = rng.standard_normal((rows, k)).astype(np.float32)
        b = rng.standard_normal((groups, n, k)).astype(np.float32)
        sa = rng.uniform(0.5, 2.0, rows).astype(np.float32)
        sb = rng.uniform(0.5, 2.0, (groups, n)).astype(np.float32)
    return f8.encode(a, ta), f8.encode(b, tb), sa, sb


def padded(u8, pitch, entry_gap=0):
    """Device copy of FP8 bytes (..., rows, cols) at `pitch` bytes per row and `entry_gap` bytes between entries, the
    padding filled with NaN bytes.  Returns (buffer, pitch, entry stride)."""
    u8 = u8.reshape((-1,) + u8.shape[-2:])
    e, r, c = u8.shape
    stride = r * pitch + entry_gap
    buf = np.full(e * stride + 16, NAN8, np.uint8)
    for i in range(e):
        buf[i * stride:i * stride + r * pitch].reshape(r, pitch)[:, :c] = u8[i]
    return dev(buf), pitch, stride


class Grouped:
    """A grouped FP8 problem: sizes (rows per group, or explicit offs), n, k, operands at padded pitches."""

    def __init__(self, ta, tb, sizes, n, k, seed, exact=False, offs=None, total_m=None):
        self.ta, self.tb, self.n, self.k = ta, tb, n, k
        self.G = len(sizes) if offs is None else len(offs)
        self.offs_list = list(np.cumsum(sizes)) if offs is None else list(offs)
        self.total_m = total_m if total_m is not None else int(sum(sizes))
        self.ends = gg.clamped_ends(self.offs_list, self.total_m)
        rng = np.random.default_rng(seed)
        self.a8, self.b8, self.sa, self.sb = operands(rng, ta, tb, self.total_m, n, k, self.G, exact)
        self.A, self.lda, _ = padded(self.a8, pad16(k) + 16)
        self.B, self.ldb, self.stride_b = padded(self.b8, pad16(k) + 32, entry_gap=48)
        self.Sa = dev(self.sa)
        sbp = np.full((self.G, n + 5), np.nan, np.float32)            # scale_b rows n + 5 apart, NaN between them
        sbp[:, :n] = self.sb
        self.Sb, self.ssb = dev(sbp), n + 5
        self.offs = torch.tensor([int(o) for o in self.offs_list], dtype=torch.int32, device="cuda")
        self.ldc = n + 8

    def c_buf(self, o):
        return torch.full((max(self.total_m, 1), self.ldc), float("nan"), dtype=f8.out_dtype(o), device="cuda")

    def call(self, gemm, C, o, fast, k=None, stream=None):
        return gemm.lib.b200_gemm_fp8_grouped(self.ta, self.tb, self.total_m, self.n, self.k if k is None else k,
                                              self.A.data_ptr(), self.lda, self.B.data_ptr(), self.ldb, self.stride_b,
                                              self.offs.data_ptr(), self.G, self.Sa.data_ptr(), self.Sb.data_ptr(),
                                              self.ssb, C.data_ptr(), self.ldc, o, fast, stream)

    def reference(self, gemm, o, fast):
        """Each group by b200_gemm_fp8 (N, T) on contiguous aligned copies of its rows, B_g and scales."""
        C = self.c_buf(o)
        lo = 0
        for g, hi in enumerate(self.ends):
            if hi > lo:
                A, lda, _ = padded(self.a8[lo:hi], pad16(self.k))
                B, ldb, _ = padded(self.b8[g], pad16(self.k))
                Sa, Sb = dev(self.sa[lo:hi]), dev(self.sb[g])
                esz = C.element_size()
                rc = gemm.lib.b200_gemm_fp8(0, 1, self.ta, self.tb, hi - lo, self.n, self.k, A.data_ptr(), lda,
                                            B.data_ptr(), ldb, Sa.data_ptr(), 1, Sb.data_ptr(), 1, None,
                                            C.data_ptr() + lo * self.ldc * esz, self.ldc, o, fast, None)
                assert rc == 0, rc
            lo = hi
        torch.cuda.synchronize()
        return C

    def oracle(self, o):
        """The numpy model rn(rn(acc * sa) * sb) rounded to the output type, NaN past the last group."""
        want = np.full((max(self.total_m, 1), self.ldc), np.nan, np.float32)
        a = f8.decode(self.a8, self.ta)
        lo = 0
        for g, hi in enumerate(self.ends):
            if hi > lo:
                b = f8.decode(self.b8[g], self.tb).T
                want[lo:hi, :self.n] = f8.oracle(a[lo:hi], b, self.sa[lo:hi], self.sb[g], None, o)
            lo = hi
        return want


def set_mode(hooks, mode):
    hooks.b200_gemm_debug_set_bn(0 if mode == "acc" else mode)
    return 0 if mode == "acc" else 1


ZIPF = [700, 300, 0, 120, 60, 1, 0, 17]                 # skewed, with empty groups; total 1198 (not a tile multiple)


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_grouped_bit_identical_to_fp8_per_group(gemm, hooks, sms, pair):
    """Every C type and mode: each group equals b200_gemm_fp8 on its own rows at the same width; n and total_m are not
    tile multiples and k is a multiple of 16 but not of 128.  Reports the kernel name and the schedule."""
    ta, tb = pair
    P = Grouped(ta, tb, ZIPF, 200, 208, seed=1)
    for o in OUTS:
        for mode in MODES:
            fast = set_mode(hooks, mode)
            C = P.c_buf(o)
            assert P.call(gemm, C, o, fast) == 0
            torch.cuda.synchronize()
            assert gemm.last_kernel() == kernel_name(ta, tb, o, "grp", mode)
            bn = 128 if mode == "acc" else mode
            assert bt.last_schedule(gemm) == gg.grp_schedule(P.total_m, P.n, P.G, bn, sms)
            ref = P.reference(gemm, o, fast)
            assert tr.same_bits(C, ref), (o, mode)


@gpu
def test_grouped_heuristic_width(gemm, hooks, sms):
    """Fast mode without a forced width takes pick_bn's width over the tile bound, as b200_gemm_bf16_grouped does."""
    for n in (4096, 1536, 640):
        P = Grouped(E4M3, E4M3, [1000, 24, 3000, 72], n, 256, seed=2)
        C = P.c_buf(OUT_BF16)
        assert P.call(gemm, C, OUT_BF16, 1) == 0
        bn = gg.grp_pick_bn(P.total_m, n, P.G, sms)
        assert gemm.last_kernel() == kernel_name(E4M3, E4M3, OUT_BF16, "grp", bn)
        hooks.b200_gemm_debug_set_bn(bn)
        assert tr.same_bits(C, P.reference(gemm, OUT_BF16, 1))
        hooks.b200_gemm_debug_set_bn(0)


@gpu
@pytest.mark.parametrize("offs", [[0, 0, 50, 50, 300], [-5, 40, 20, 600, 900], [128, 256, 384, 512, 513],
                                  [3, 2, 1, 0, -1], [700, 800, 900, 1000, 1100]],
                         ids=["empty", "negative-and-too-large", "tile-aligned", "non-monotone", "past-the-end"])
def test_grouped_clamped_offsets(gemm, hooks, offs):
    """Offsets are clamped as b200_gemm_bf16_grouped's, on the device; rows at or after end_{G-1} stay NaN."""
    P = Grouped(E4M3, E5M2, None, 136, 144, seed=3, offs=offs, total_m=620)
    for mode in ("acc", 128):
        fast = set_mode(hooks, mode)
        C = P.c_buf(OUT_F32)
        assert P.call(gemm, C, OUT_F32, fast) == 0
        torch.cuda.synchronize()
        assert tr.same_bits(C, P.reference(gemm, OUT_F32, fast)), mode
        assert bool(torch.isnan(C[P.ends[-1]:]).all()) and bool(torch.isnan(C[:, P.n:]).all())


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_grouped_exact_oracle(gemm, hooks, pair):
    """Integer operands and power-of-two scales: every C type and mode equals the numpy model bit for bit."""
    ta, tb = pair
    P = Grouped(ta, tb, [130, 0, 257, 1, 90], 150, 400, seed=4, exact=True)
    for o in OUTS:
        want = torch.from_numpy(P.oracle(o))
        for mode in ("acc", 256, 128):
            fast = set_mode(hooks, mode)
            C = P.c_buf(o)
            assert P.call(gemm, C, o, fast) == 0
            torch.cuda.synchronize()
            assert tr.same_bits(C.float().cpu(), want), (o, mode)


@gpu
def test_grouped_k_zero(gemm):
    """k == 0: +0 over rows [0, end_{G-1}) through fill_zero_grp, no scale or operand read (null scales refused
    first, so NaN scales stand in), rows after the last group untouched."""
    P = Grouped(E4M3, E4M3, [40, 0, 100], 64, 32, seed=5)
    P.Sa.fill_(float("nan"))
    for o in OUTS:
        C = P.c_buf(o)
        assert P.call(gemm, C, o, 0, k=0) == 0
        torch.cuda.synchronize()
        assert gemm.last_kernel() == "fill_zero_grp"
        assert bool((C[:140, :64].float() == 0).all()) and not bool(torch.signbit(C[:140, :64].float()).any())
        assert bool(torch.isnan(C[:, 64:]).all())


# ==== batched ======================================================================================================
class Batched:
    def __init__(self, ta, tb, batch, m, n, k, seed, exact=False, broadcast_a=False):
        self.ta, self.tb, self.batch, self.m, self.n, self.k = ta, tb, batch, m, n, k
        rng = np.random.default_rng(seed)
        a8, self.b8, _, self.sb = operands(rng, ta, tb, m, n, k, batch, exact)
        self.a8 = np.broadcast_to(a8, (batch, m, k)) if broadcast_a else \
            operands(rng, ta, tb, batch * m, 1, k, 1, exact)[0].reshape(batch, m, k)
        sa = operands(rng, ta, tb, batch * m, 1, 1, 1, exact)[2].reshape(batch, m)
        self.sa = sa
        self.A, self.lda, self.stride_a = padded(a8 if broadcast_a else self.a8, pad16(k) + 16, entry_gap=32)
        if broadcast_a:
            self.stride_a = 0
        self.B, self.ldb, self.stride_b = padded(self.b8, pad16(k), entry_gap=16)
        sap = np.full((batch, m + 3), np.nan, np.float32)
        sap[:, :m] = sa
        self.Sa, self.ssa = dev(sap), m + 3
        self.Sb, self.ssb = dev(self.sb), n
        self.ldc = n + 8
        self.stride_c = (m + 1) * self.ldc

    def c_buf(self, o):
        return torch.full((self.batch * (self.m + 1), self.ldc), float("nan"), dtype=f8.out_dtype(o), device="cuda")

    def call(self, gemm, C, o, fast, k=None):
        return gemm.lib.b200_gemm_fp8_batched(self.ta, self.tb, self.m, self.n, self.k if k is None else k,
                                              self.A.data_ptr(), self.lda, self.stride_a, self.B.data_ptr(), self.ldb,
                                              self.stride_b, self.Sa.data_ptr(), self.ssa, self.Sb.data_ptr(), self.ssb,
                                              C.data_ptr(), self.ldc, self.stride_c, self.batch, o, fast, None)

    def reference(self, gemm, o, fast):
        C = self.c_buf(o)
        esz = C.element_size()
        for e in range(self.batch):
            A, lda, _ = padded(np.ascontiguousarray(self.a8[e]), pad16(self.k))
            B, ldb, _ = padded(self.b8[e], pad16(self.k))
            Sa, Sb = dev(self.sa[e]), dev(self.sb[e])
            rc = gemm.lib.b200_gemm_fp8(0, 1, self.ta, self.tb, self.m, self.n, self.k, A.data_ptr(), lda, B.data_ptr(),
                                        ldb, Sa.data_ptr(), 1, Sb.data_ptr(), 1, None,
                                        C.data_ptr() + e * self.stride_c * esz, self.ldc, o, fast, None)
            assert rc == 0, rc
        torch.cuda.synchronize()
        return C

    def oracle(self, o):
        want = np.full((self.batch * (self.m + 1), self.ldc), np.nan, np.float32)
        for e in range(self.batch):
            r0 = e * (self.m + 1)
            want[r0:r0 + self.m, :self.n] = f8.oracle(f8.decode(np.ascontiguousarray(self.a8[e]), self.ta),
                                                       f8.decode(self.b8[e], self.tb).T, self.sa[e], self.sb[e], None, o)
        return want


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
@pytest.mark.parametrize("broadcast_a", [False, True], ids=["strided", "broadcast-A"])
def test_batched_bit_identical_to_fp8_per_entry(gemm, hooks, sms, pair, broadcast_a):
    """Every C type and mode: each entry equals its own b200_gemm_fp8 call, with a broadcast A (stride 0) scaled by
    each entry's own scale_a; the gap rows between entries of C stay NaN."""
    ta, tb = pair
    P = Batched(ta, tb, 4, 300, 200, 208, seed=6, broadcast_a=broadcast_a)
    for o in OUTS:
        for mode in MODES:
            fast = set_mode(hooks, mode)
            C = P.c_buf(o)
            assert P.call(gemm, C, o, fast) == 0
            torch.cuda.synchronize()
            assert gemm.last_kernel() == kernel_name(ta, tb, o, "bat", mode)
            bn = 128 if mode == "acc" else mode
            tiles = 4 * 3 * -(-200 // bn)
            assert bt.last_schedule(gemm) == (tiles, 1, tiles, min(tiles, sms))
            assert tr.same_bits(C, P.reference(gemm, o, fast)), (o, mode)


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_batched_exact_oracle(gemm, hooks, pair):
    ta, tb = pair
    P = Batched(ta, tb, 3, 130, 150, 400, seed=7, exact=True)
    for o in OUTS:
        want = torch.from_numpy(P.oracle(o))
        for mode in ("acc", 192):
            fast = set_mode(hooks, mode)
            C = P.c_buf(o)
            assert P.call(gemm, C, o, fast) == 0
            torch.cuda.synchronize()
            assert tr.same_bits(C.float().cpu(), want), (o, mode)


@gpu
def test_batch_of_one_is_the_fp8_call(gemm, hooks):
    """batch == 1 is the (N, T) b200_gemm_fp8 call: same kernel name and bits; k == 0 of a batch is fill_zero_bat."""
    P = Batched(E4M3, E4M3, 1, 300, 200, 208, seed=8)
    for mode in ("acc", 256):
        fast = set_mode(hooks, mode)
        C = P.c_buf(OUT_BF16)
        assert P.call(gemm, C, OUT_BF16, fast) == 0
        name = gemm.last_kernel()
        assert name == ("tc_e4m3_obf16_acc_128x128" if mode == "acc" else "tc_e4m3_obf16_128x256")
        assert tr.same_bits(C, P.reference(gemm, OUT_BF16, fast))
    Q = Batched(E4M3, E4M3, 3, 20, 40, 32, seed=9)
    Q.Sa.fill_(float("nan"))
    C = Q.c_buf(OUT_F32)
    assert Q.call(gemm, C, OUT_F32, 0, k=0) == 0
    torch.cuda.synchronize()
    assert gemm.last_kernel() == "fill_zero_bat"
    for e in range(3):
        blk = C[e * 21:e * 21 + 21]
        assert bool((blk[:20, :40] == 0).all()) and bool(torch.isnan(blk[20]).all()) and bool(torch.isnan(blk[:, 40:]).all())


# ==== CUDA graph: offsets and scales rewritten on the device between replays ======================================
@gpu
def test_cuda_graph_replay_with_new_offsets_and_scales(gemm, hooks):
    """One captured grouped call (a host synchronisation inside it would fail the capture); offs and both scales are
    rewritten in place between replays, and each replay equals the per-group b200_gemm_fp8 calls for the new values."""
    P = Grouped(E4M3, E4M3, [125] * 8, 256, 192, seed=10)
    hooks.b200_gemm_debug_set_bn(128)
    C = P.c_buf(OUT_BF16)
    assert P.call(gemm, C, OUT_BF16, 1) == 0                          # tensor maps and kernel attributes set up first
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                                     # captures torch's current (side) stream
        assert P.call(gemm, C, OUT_BF16, 1, stream=torch.cuda.current_stream().cuda_stream) == 0
    rng = np.random.default_rng(11)
    for offs in ([600, 600, 700, 700, 900, 990, 1000, 1000], [0, 10, 20, 30, 40, 50, 60, 900]):
        C.fill_(float("nan"))
        P.offs.copy_(torch.tensor(offs, dtype=torch.int32))
        P.sa = rng.uniform(0.25, 4.0, P.total_m).astype(np.float32)
        P.sb = rng.uniform(0.25, 4.0, (P.G, P.n)).astype(np.float32)
        P.Sa.copy_(torch.from_numpy(P.sa))
        P.Sb[:, :P.n].copy_(torch.from_numpy(P.sb))
        graph.replay()
        torch.cuda.synchronize()
        P.ends = gg.clamped_ends(offs, P.total_m)
        assert tr.same_bits(C, P.reference(gemm, OUT_BF16, 1)), offs
        assert bool(torch.isnan(C[P.ends[-1]:]).all())


# ==== MoE shapes: scaled_grouped_mm against float64 and torch._scaled_grouped_mm ==================================
def rowwise_fp8(x, dim):
    """Rowwise e4m3 quantisation along `dim` (the reduction dimension): q = x / s, s = amax / 448."""
    s = (x.abs().amax(dim=dim, keepdim=True).float() / 448.0).clamp(min=1e-12)
    return (x / s).to(torch.float8_e4m3fn), s.squeeze(dim)


# Fast accumulation (one tensor-core accumulator over K) has no derived bound: its class, error over sum |a b| sa sb,
# measured on these operands on an H100 80GB HBM3 (DESIGN §9), with margin.
FAST_CLASS = 2.0 ** -9


@gpu
@pytest.mark.parametrize("form", ["2d-3d", "3d-3d"])
def test_moe_shapes_against_torch(gemm, form):
    """An MoE up-projection: promoted within (8 * 2^-13 + ceil(k / 128) * 2^-24) * sum|a b| * sa * sb of the exact
    result (fp32 out), fast within FAST_CLASS of the same sum; bf16 out against torch._scaled_grouped_mm within twice the bound
    plus one bf16 rounding of each.  Where torch refuses the call on this stack the comparison with it skips."""
    g = torch.Generator(device="cuda").manual_seed(12)
    G, d, dff = 8, 1024, 2048
    if form == "2d-3d":
        sizes = [1200, 40, 0, 700, 300, 1, 1500, 355]
        offs = torch.tensor(np.cumsum(sizes), dtype=torch.int32, device="cuda")
        x = torch.randn((sum(sizes), d), device="cuda", generator=g)
    else:
        offs, x = None, torch.randn((G, 512, d), device="cuda", generator=g)
    W = torch.randn((G, dff, d), device="cuda", generator=g)
    xq, sa = rowwise_fp8(x, -1)
    Wq, sb = rowwise_fp8(W, -1)                                       # (G, dff) scales of the columns of B
    B = Wq.transpose(-2, -1)
    xd, Bd = xq.double(), B.double()
    if offs is None:
        exact = (xd @ Bd) * sa.double()[..., None] * sb.double()[:, None, :]
        mag = (xd.abs() @ Bd.abs()) * sa.double()[..., None] * sb.double()[:, None, :]
    else:
        ends = [0] + offs.tolist()
        exact = torch.cat([(xd[ends[i]:ends[i + 1]] @ Bd[i]) for i in range(G)])
        mag = torch.cat([(xd[ends[i]:ends[i + 1]].abs() @ Bd[i].abs()) for i in range(G)])
        sbr = torch.cat([sb[i].double().expand(ends[i + 1] - ends[i], dff) for i in range(G)])
        exact, mag = exact * sa.double()[:, None] * sbr, mag * sa.double()[:, None] * sbr
    bound = (8 * 2.0 ** -13 + math.ceil(d / 128) * 2.0 ** -24) * mag + 2.0 ** -22 * exact.abs()
    for fast in (False, True):
        y32 = gemm.scaled_grouped_mm(xq, B, sa, sb, offs, out_dtype=torch.float32, use_fast_accum=fast)
        err = (y32.double() - exact).abs()
        ratio = float(((err - 2.0 ** -22 * exact.abs()) / mag).max())        # error over sum |a b| sa sb
        print(f"{form} use_fast_accum={fast}: max error / sum|a b| sa sb = {ratio:.3e}")
        assert bool((err <= (FAST_CLASS * mag + 2.0 ** -22 * exact.abs() if fast else bound)).all()), (fast, ratio)
        y = gemm.scaled_grouped_mm(xq, B, sa, sb, offs, use_fast_accum=fast)
        assert y.dtype == torch.bfloat16 and ("_grp_" if offs is not None else "_bat_") in gemm.last_kernel()
        try:
            t = torch._scaled_grouped_mm(xq, B, sa, sb, offs=offs, out_dtype=torch.bfloat16, use_fast_accum=fast)
        except (RuntimeError, NotImplementedError) as e:
            pytest.skip(f"torch._scaled_grouped_mm refuses this call here: {e}")
        tol = 2 * (FAST_CLASS * mag if fast else bound) + 2.0 ** -8 * (exact.abs() + t.double().abs())
        assert bool(((y.double() - t.double()).abs() <= tol).all()), fast
