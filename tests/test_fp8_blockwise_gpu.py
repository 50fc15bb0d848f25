"""Blockwise-scaled FP8 GEMMs (b200_gemm_fp8_blockwise) and scaled_mm() with torch._scaled_mm's 1 x 128 / 128 x 128
scales.  With q = ceil(k / 128) k-blocks, block b covering K elements [128 b, 128 b + 128):

    s_b(i, j) = rn(sa_b(i) * sb_b(j));   sum = fma(acc_b(i, j), s_b(i, j), sum) for b = 0 .. q - 1, from sum = +0;
    C = round_out(rn(sum + bias_j))

acc_b is the FP8 product over block b.  The oracle decodes the operands with torch's CPU casts, forms each acc_b in
float64 (exact, and exact in fp32, on the integer operands used here) and applies the chain of fp32 FMAs exactly:
numpy has no fp32 FMA, so each one is the exact float64 product, a float64 TwoSum with the addend, a round to odd, and
one cast to float32 (float64 carries more than 24 + 2 bits, so that cast is the single correct rounding).  On such
operands the whole chain is determined, so every recipe, pair, C type, layout, scale layout and tail must equal the
oracle bit for bit.  On random operands the result must stay inside the bound derived in rel_bound() from the header's
per-128-element chunk bound.

The argument checks, scaled_mm's recipe resolution and refusals, and the oracle itself need no GPU."""
import math
from fractions import Fraction

import numpy as np
import pytest

from test_fp8_gpu import (E4M3, E5M2, OP_N, OP_T, OUT_BF16, OUT_F16, OUT_F32, OUT_NAME, PAIR_NAME, PAIRS, _has_gpu,
                          decode, encode, exact_operands, fp8_dtype, oracle, out_dtype, round_out, same_bits)

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")
# (scale_a_block, scale_b_block): torch's three recipes
RECIPES = [(1, 128), (1, 1), (128, 1)]
RECIPE_NAME = {(1, 128): "1x128-128x128", (1, 1): "1x128-1x128", (128, 1): "128x128-1x128"}
INT64_MAX = 2 ** 63 - 1
MAX_INDEX = INT64_MAX // 4   # the last scale's byte offset must fit a signed 64-bit integer


def cdiv(a, b):
    return -(-a // b)


def same_bits_or_nan(x, y):
    """NaN at the same places (any payload) and the same bits everywhere else."""
    nan = np.isnan(x)
    return np.array_equal(nan, np.isnan(y)) and same_bits(np.where(nan, 0, x).astype(np.float32),
                                                         np.where(nan, 0, y).astype(np.float32))


# ==== the oracle ===================================================================================================
def fma32(x, y, z):
    """Exact fp32 fused multiply-add rn(x * y + z) of float32 arrays, IEEE non-finite rules included."""
    x, y, z = (np.asarray(v, np.float32).astype(np.float64) for v in (x, y, z))
    with np.errstate(invalid="ignore", over="ignore"):
        p = x * y                                   # exact: 48 significant bits, exponent inside float64's range
        s = p + z
        bp = s - z                                  # TwoSum: s + err == p + z exactly
        err = (p - (s - bp)) + (z - bp)
        finite = np.isfinite(s)
        odd_step = finite & (err != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(odd_step, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def expand_scales(sa, sb, blocks, m, n):
    """The recipe's scale tensors (numpy) -> per-row sa_full (m, q) and per-column sb_full (q, n), float32."""
    a_blk, b_blk = blocks
    sa_full = np.repeat(sa, 128, axis=0)[:m] if a_blk == 128 else sa
    sb_full = np.repeat(sb, 128, axis=1)[:, :n] if b_blk == 128 else sb
    return np.asarray(sa_full, np.float32), np.asarray(sb_full, np.float32)


def block_sums(a, b, sa_full, sb_full, two_roundings=False):
    """The fp32 running sum after every k-block.  two_roundings: rn(rn(acc * s) + sum) instead of the FMA."""
    m, k = a.shape
    s = np.zeros((m, b.shape[1]), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for kb in range(cdiv(k, 128)):
            sl = slice(128 * kb, 128 * kb + 128)
            acc = (a[:, sl].astype(np.float64) @ b[sl].astype(np.float64)).astype(np.float32)
            sc = sa_full[:, kb][:, None] * sb_full[kb][None, :]
            s = (acc * sc + s).astype(np.float32) if two_roundings else fma32(acc, sc, s)
    return s


def oracle_blockwise(a, b, sa_full, sb_full, bias, o, two_roundings=False):
    s = block_sums(a, b, sa_full, sb_full, two_roundings)
    with np.errstate(invalid="ignore", over="ignore"):
        if bias is not None:
            s = (s + bias[None, :].astype(np.float32)).astype(np.float32)
    return round_out(s, o)


def fraction_to_f32(f):
    """Round a Fraction to the nearest float32 (ties to even), subnormals included; finite results only."""
    if f == 0:
        return np.float32(0.0)
    e = max(math.floor(math.log2(abs(f))), -126)
    if Fraction(2) ** e > abs(f):               # log2 rounded up near a power of two
        e -= 1
    elif Fraction(2) ** (e + 1) <= abs(f):
        e += 1
    e = max(e, -126)
    ulp = Fraction(2) ** (e - 23)
    r = round(f / ulp) * ulp                    # Python rounds a Fraction half to even
    return np.float32(float(r))


def test_oracle_fma_matches_exact_rationals():
    """fma32 equals the exactly rounded rational x * y + z on crafted near-cancelling cases, ties and subnormals."""
    rng = np.random.default_rng(11)
    n = 4000
    x = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    y = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    p32 = (x.astype(np.float64) * y.astype(np.float64)).astype(np.float32)
    pert = rng.integers(-3, 4, n).astype(np.float32) * np.spacing(np.abs(p32)) * rng.choice([1, 2 ** -12, 2 ** -23], n)
    z = np.where(rng.random(n) < 0.7, -p32 + pert.astype(np.float32), rng.standard_normal(n)).astype(np.float32)
    # small magnitudes: results in the subnormal range
    x[:200] = (rng.standard_normal(200) * 2.0 ** -70).astype(np.float32)
    y[:200] = (rng.standard_normal(200) * 2.0 ** -70).astype(np.float32)
    z[:200] = (rng.standard_normal(200) * 2.0 ** -140).astype(np.float32)
    got = fma32(x, y, z)
    for i in range(n):
        want = fraction_to_f32(Fraction(float(x[i])) * Fraction(float(y[i])) + Fraction(float(z[i])))
        assert got[i] == want and np.signbit(got[i]) == np.signbit(want) or (got[i] == 0 and want == 0), \
            (i, x[i], y[i], z[i], got[i], want)
    # IEEE: 0 * inf is NaN, inf propagates, the sign of an exact zero follows round to nearest
    assert np.isnan(fma32(0.0, np.inf, 1.0)) and fma32(1.0, np.inf, 1.0) == np.inf
    assert not np.signbit(fma32(-0.0, 1.0, 0.0)) and np.signbit(fma32(-0.0, 1.0, -0.0))


@need_torch
def test_oracle_with_power_of_two_scales_is_the_scaled_product():
    """Constant power-of-two scales on exact operands: the FMA chain is the plain scaled product of test_fp8_gpu."""
    rng = np.random.default_rng(12)
    m, n, k = 40, 56, 401
    for ta, tb in PAIRS:
        a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        a, b = decode(a8, ta), decode(b8, tb)
        q = cdiv(k, 128)
        for s_a, s_b in ((1.0, 1.0), (0.25, 8.0), (2.0 ** -5, 2.0 ** 3)):
            for o in (OUT_F32, OUT_BF16, OUT_F16):
                got = oracle_blockwise(a, b, np.full((m, q), s_a, np.float32), np.full((q, n), s_b, np.float32), None, o)
                want = oracle(a, b, np.full(m, s_a, np.float32), np.full(n, s_b, np.float32), None, o)
                assert same_bits(got, want), (ta, tb, s_a, s_b, o)


# ==== the C ABI through ctypes =====================================================================================
def call(gemm, op_a=OP_N, op_b=OP_T, ta=E4M3, tb=E4M3, m=4, n=4, k=4, a=1, lda=None, b=1, ldb=None, sa=1, a_blk=1,
         sa_row=None, sa_kb=None, sb=1, b_blk=128, sb_kb=None, sb_col=None, bias=None, c=1, ldc=None, out=OUT_BF16,
         stream=None):
    """b200_gemm_fp8_blockwise with raw pointers (ints; 1 stands for a dummy non-null pointer where no GPU is present).
    Default strides: contiguous (rows, q) scale_a and (q, cols) scale_b."""
    lda = lda if lda is not None else (m if op_a else k)
    ldb = ldb if ldb is not None else (k if op_b else n)
    ldc = ldc if ldc is not None else n
    q = cdiv(k, 128)
    sa_row = sa_row if sa_row is not None else q
    sa_kb = sa_kb if sa_kb is not None else 1
    sb_kb = sb_kb if sb_kb is not None else (cdiv(n, 128) if b_blk == 128 else n)
    sb_col = sb_col if sb_col is not None else 1
    return gemm.lib.b200_gemm_fp8_blockwise(op_a, op_b, ta, tb, m, n, k, a, lda, b, ldb, sa, a_blk, sa_row, sa_kb, sb,
                                            b_blk, sb_kb, sb_col, bias, c, ldc, out, stream)


def test_blockwise_argument_validation(gemm):
    """Refusals before the device is touched, each at its exact bound: they hold with or without a GPU."""
    assert call(gemm, ta=2) == -1 and call(gemm, tb=-1) == -1
    assert call(gemm, out=3) == -1 and call(gemm, out=-1) == -1
    for bad in (0, 2, 64, 127, 129, 256, -1, -128):
        assert call(gemm, a_blk=bad) == -1 and call(gemm, b_blk=bad) == -1
    for name in ("sa_row", "sa_kb", "sb_kb", "sb_col"):
        assert call(gemm, **{name: -1}) == -1
    assert call(gemm, op_a=2) == -1 and call(gemm, op_b=-1) == -1
    assert call(gemm, m=-1) == -1 and call(gemm, n=-1) == -1 and call(gemm, k=-1) == -1
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            m, n, k = 5, 6, 7
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, lda=(m if op_a else k) - 1) == -1
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, ldb=(k if op_b else n) - 1) == -1
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, ldc=n - 1) == -1
    assert call(gemm, a=None) == -1 and call(gemm, b=None) == -1 and call(gemm, c=None) == -1
    assert call(gemm, sa=None) == -1 and call(gemm, sb=None) == -1          # a null scale with work to do
    assert call(gemm, sa=None, k=0) == -1 and call(gemm, sb=None, k=0) == -1
    # (128, 128) is not a torch recipe; e5m2 x e5m2 is not supported: -3 whatever the shape
    assert call(gemm, a_blk=128, b_blk=128) == -3 and call(gemm, a_blk=128, b_blk=128, m=0) == -3
    assert call(gemm, ta=E5M2, tb=E5M2) == -3 and call(gemm, ta=E5M2, tb=E5M2, n=0) == -3
    # m == 0 or n == 0: a no-op, null pointers included
    assert call(gemm, m=0, a=None, b=None, c=None, sa=None, sb=None) == 0
    assert call(gemm, n=0, a=None, b=None, c=None, sa=None, sb=None) == 0
    # the last scale index one past the bound: (rows - 1) * row_stride + (q - 1) * kb_stride > (2^63 - 1) / 4
    assert call(gemm, m=2, sa_row=MAX_INDEX + 1, sa_kb=0) == -1
    assert call(gemm, m=2, k=129, sa_row=0, sa_kb=MAX_INDEX + 1) == -1
    assert call(gemm, m=2, k=129, sa_row=MAX_INDEX // 2, sa_kb=MAX_INDEX // 2 + 2) == -1
    assert call(gemm, m=129, a_blk=128, b_blk=1, sa_row=MAX_INDEX + 1, sa_kb=0) == -1
    assert call(gemm, n=2, b_blk=1, sb_col=MAX_INDEX + 1, sb_kb=0) == -1
    assert call(gemm, n=129, b_blk=128, sb_col=MAX_INDEX + 1, sb_kb=0) == -1
    assert call(gemm, k=129, sb_kb=MAX_INDEX + 1) == -1
    assert call(gemm, m=3, sa_row=INT64_MAX, sa_kb=0) == -1                 # overflows 64 bits outright


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_blockwise_accepts_at_the_bounds_without_device(gemm):
    """Every accepted recipe x pair x C type, the smallest legal ld, stride 0, k == 0 with null operands and the last
    scale index exactly at its bound reach the device check (-2)."""
    for blocks in RECIPES:
        for ta, tb in PAIRS:
            for o in (OUT_F32, OUT_BF16, OUT_F16):
                assert call(gemm, ta=ta, tb=tb, a_blk=blocks[0], b_blk=blocks[1], out=o) == -2
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            assert call(gemm, op_a, op_b, m=5, n=6, k=7) == -2
    assert call(gemm, k=0, a=None, b=None) == -2
    assert call(gemm, sa_row=0, sa_kb=0, sb_kb=0, sb_col=0) == -2
    assert call(gemm, m=2, sa_row=MAX_INDEX, sa_kb=0) == -2
    assert call(gemm, m=2, k=129, sa_row=0, sa_kb=MAX_INDEX) == -2
    assert call(gemm, m=2, k=129, sa_row=MAX_INDEX // 2, sa_kb=MAX_INDEX // 2 + 1) == -2
    assert call(gemm, m=129, a_blk=128, b_blk=1, sa_row=MAX_INDEX, sa_kb=0) == -2
    assert call(gemm, m=128, a_blk=128, b_blk=1, sa_row=INT64_MAX, sa_kb=0) == -2   # one row block: stride unused
    assert call(gemm, n=2, b_blk=1, sb_col=MAX_INDEX, sb_kb=0) == -2
    assert call(gemm, n=129, b_blk=128, sb_col=MAX_INDEX, sb_kb=0) == -2
    assert call(gemm, k=129, sb_kb=MAX_INDEX) == -2


# ==== scaled_mm: recipe resolution and refusals (CPU) ==============================================================
def _fp8(shape, t=E4M3, device="cpu"):
    return torch.zeros(shape, dtype=torch.float32, device=device).to(fp8_dtype(t))


@need_torch
def test_scaled_mm_resolves_blockwise_recipes(gemm):
    """The three recipes resolve from the scales' shapes; the k <= 128 shapes that are also tensorwise / rowwise keep
    that meaning (use_fast_accum is accepted for them, refused for a blockwise recipe)."""
    m, n, k = 200, 300, 401
    q, mb, nb = 4, 2, 3
    ones = torch.ones
    assert gemm._blockwise_recipe(ones(m, q), ones(q, nb), m, n, k) == (1, 128)
    assert gemm._blockwise_recipe(ones(m, q), ones(q, n), m, n, k) == (1, 1)
    assert gemm._blockwise_recipe(ones(mb, q), ones(q, n), m, n, k) == (128, 1)
    assert gemm._blockwise_recipe(ones(q, m).t(), ones(nb, q).t(), m, n, k) == (1, 128)   # strides do not matter
    assert gemm._blockwise_recipe(ones(mb, q), ones(q, nb), m, n, k) is None               # (128, 128)
    assert gemm._blockwise_recipe(ones(m, q), ones(nb, q), m, n, k) is None
    assert gemm._blockwise_recipe(ones(m, q).double(), ones(q, nb), m, n, k) is None
    assert gemm._blockwise_recipe(ones(m * q), ones(q, nb), m, n, k) is None
    A, B = _fp8((m, k)), _fp8((k, n))
    for sa, sb in ((ones(m, q), ones(q, nb)), (ones(m, q), ones(q, n)), (ones(mb, q), ones(q, n))):
        with pytest.raises(ValueError, match="CUDA"):                 # resolved; the CPU tensors are refused next
            gemm.scaled_mm(A, B, sa, sb)
        with pytest.raises(ValueError, match="use_fast_accum"):
            gemm.scaled_mm(A, B, sa, sb, use_fast_accum=True)
    # k <= 128: (m, 1) with (1, 1) or (1, n) are rowwise / tensorwise shapes too, and stay so
    A, B = _fp8((m, 100)), _fp8((100, n))
    assert gemm._blockwise_recipe(ones(m, 1), ones(1, 1), m, 128, 100) == (1, 128)
    for sa, sb in ((ones(m, 1), ones(1, 1)), (ones(m, 1), ones(1, n)), (ones(1, 1), ones(1, n))):
        with pytest.raises(ValueError, match="CUDA"):
            gemm.scaled_mm(A, B, sa, sb, use_fast_accum=True)
    # off the tensorwise / rowwise shapes, the same k takes the blockwise recipes
    with pytest.raises(ValueError, match="use_fast_accum"):
        gemm.scaled_mm(A, B, ones(m, 1), ones(1, nb), use_fast_accum=True)


@need_torch
def test_scaled_mm_blockwise_refusals(gemm):
    m, n, k = 200, 300, 401
    q, mb, nb = 4, 2, 3
    A, B = _fp8((m, k)), _fp8((k, n))
    ones = torch.ones
    bad = [
        (ones(m, q), ones(q, nb + 1)),            # wrong shapes
        (ones(m, q + 1), ones(q + 1, nb)),
        (ones(m + 1, q), ones(q, n)),
        (ones(mb, q), ones(q, nb)),               # (128 x 128, 128 x 128) is not a recipe
        (ones(m * q), ones(q * nb)),              # 1-D scales
        (ones(m, q), ones(q, nb, 1)),
        (ones(m, q), ones(1)),                    # mixed blockwise / tensorwise
        (ones(1), ones(q, nb)),
        (ones(m, 1), ones(q, nb)),                # mixed blockwise / rowwise
        (ones(m, q), ones(1, n)),
        (ones(m, q).double(), ones(q, nb)),       # not float32
        (ones(m, q), ones(q, nb).half()),
    ]
    for sa, sb in bad:
        with pytest.raises(ValueError):
            gemm.scaled_mm(A, B, sa, sb)
    with pytest.raises(ValueError, match="use_fast_accum"):
        gemm.scaled_mm(A, B, ones(m, q), ones(q, nb), use_fast_accum=True)
    with pytest.raises(ValueError, match="CUDA"):
        gemm.scaled_mm(A, B, ones(m, q), ones(q, nb))                        # CPU tensors


# ==== GPU ==========================================================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def strides_of(t):
    return t.stride(0), t.stride(1)


def run(gemm, a8, b8, ta, tb, Sa, Sb, blocks, bias, o, op_a=OP_N, op_b=OP_T, m=None, n=None, k=None, stream=None):
    """b200_gemm_fp8_blockwise on device copies: a8 / b8 the stored bytes (A as given by op_a, B by op_b); Sa / Sb 2-D
    float32 CUDA tensors passed with their own strides; bias float32 values of the output type, or None."""
    if m is None:
        m, k = (a8.shape[1], a8.shape[0]) if op_a else a8.shape
        n = b8.shape[0] if op_b else b8.shape[1]
    A, B = dev(a8), dev(b8)
    Bi = torch.from_numpy(bias).to(out_dtype(o)).cuda() if bias is not None else None
    Cm = torch.full((max(m, 1), max(n, 1)), float("nan"), dtype=out_dtype(o), device="cuda")
    rc = gemm.lib.b200_gemm_fp8_blockwise(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), a8.shape[1], B.data_ptr(),
                                          b8.shape[1], Sa.data_ptr(), blocks[0], *strides_of(Sa), Sb.data_ptr(),
                                          blocks[1], *strides_of(Sb), Bi.data_ptr() if Bi is not None else None,
                                          Cm.data_ptr(), max(n, 1), o, stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return Cm[:m, :n].float().cpu().numpy()


def random_scales(rng, shape):
    """fp32 scales with random significands in [2^-3, 2^3): their products round."""
    return (rng.uniform(1, 2, shape) * 2.0 ** rng.integers(-3, 3, shape)).astype(np.float32)


def recipe_scales(rng, blocks, m, n, k, make=random_scales):
    q = cdiv(k, 128)
    sa = make(rng, (m if blocks[0] == 1 else cdiv(m, 128), q))
    sb = make(rng, (q, n if blocks[1] == 1 else cdiv(n, 128)))
    return sa, sb


@gpu
@pytest.mark.parametrize("blocks", RECIPES, ids=lambda b: RECIPE_NAME[b])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
@pytest.mark.parametrize("o", [OUT_F32, OUT_BF16, OUT_F16], ids=lambda o: OUT_NAME[o])
def test_exact_class_bit_exact(gemm, blocks, pair, o):
    """Integer operands in [-2, 2] make every acc_b exact, so random fp32 scales pin rn(sa * sb), the FMA and the block
    order: every recipe, pair and C type equals the FMA oracle bit for bit, with M / N / K tails and k < 128, with and
    without a bias.  A two-rounding oracle differs on the same data, so the test discriminates."""
    ta, tb = pair
    rng = np.random.default_rng(hash((blocks, pair, o)) & 0xFFFF)
    for m, n, k in ((200, 300, 3 * 128 + 17), (64, 40, 100), (129, 257, 256)):
        a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        a, b = decode(a8, ta), decode(b8, tb)
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        sa_full, sb_full = expand_scales(sa, sb, blocks, m, n)
        if k > 128:
            fma_sum = block_sums(a, b, sa_full, sb_full)
            assert not same_bits(fma_sum, block_sums(a, b, sa_full, sb_full, two_roundings=True))
        for with_bias in (False, True):
            bias = round_out(rng.integers(-64, 65, n).astype(np.float32) / 8, o) if with_bias else None
            got = run(gemm, a8, np.ascontiguousarray(b8.T), ta, tb, dev(sa), dev(sb), blocks, bias, o)
            want = oracle_blockwise(a, b, sa_full, sb_full, bias, o)
            assert same_bits(got, want), (m, n, k, with_bias)
            assert gemm.last_kernel() == f"tc_{PAIR_NAME[pair]}_{OUT_NAME[o]}_blk_128x128"


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
def test_unit_scales_match_the_promoted_kernel(gemm, pair):
    """All block scales 1.0 on random (inexact) operands: bit for bit the promoted b200_gemm_fp8 (fast_accum = 0) with
    unit tensorwise scales, but for the sign of an exact zero (fma(acc, 1, +0) is +0 where the promoted sum is acc)."""
    ta, tb = pair
    rng = np.random.default_rng(21)
    m, n, k = 256, 384, 1000
    a8 = encode(rng.standard_normal((m, k)) * 4, ta)
    bt8 = encode(rng.standard_normal((n, k)) * 4, tb)
    q = cdiv(k, 128)
    one = torch.ones(1, device="cuda")
    for o in (OUT_F32, OUT_BF16):
        for blocks in RECIPES:
            sa, sb = recipe_scales(rng, blocks, m, n, k, lambda r, s: np.ones(s, np.float32))
            got = run(gemm, a8, bt8, ta, tb, dev(sa), dev(sb), blocks, None, o)
            A, Bt = dev(a8), dev(bt8)
            Cm = torch.empty((m, n), dtype=out_dtype(o), device="cuda")
            assert gemm.lib.b200_gemm_fp8(OP_N, OP_T, ta, tb, m, n, k, A.data_ptr(), k, Bt.data_ptr(), k, one.data_ptr(),
                                          0, one.data_ptr(), 0, None, Cm.data_ptr(), n, o, 0, None) == 0
            ref = Cm.float().cpu().numpy()
            assert np.array_equal(got, ref), (o, blocks)
            assert q > 1 and not np.isnan(got).any()


def rel_bound(k):
    """Per element: |C - exact| <= w * (8 * 2^-13 + 2 * 2^-24) + q * 2^-24 * w, w = sum_b |s_b| sum_{k in b} |a_k b_k|.
    8 * 2^-13 bounds the tensor core's error on one 128-element block (the header's chunk bound); 2^-24 the rounding of
    s_b times |acc_b| <= sum |a b|, and once more each FMA's rounding of the block's term; q * 2^-24 * w the roundings
    of the running sum, each at most 2^-24 of a partial sum bounded by w.  Returns the factor of w."""
    return 8 * 2.0 ** -13 + 2 * 2.0 ** -24 + cdiv(k, 128) * 2.0 ** -24 * 1.01


def exact_and_weight(a, b, sa_full, sb_full):
    """float64: sum_b sa sb (a_b @ b_b) of the decoded operands, and w = sum_b |rn(sa sb)| (|a_b| @ |b_b|)."""
    ex = np.zeros((a.shape[0], b.shape[1]))
    w = np.zeros_like(ex)
    for kb in range(cdiv(a.shape[1], 128)):
        sl = slice(128 * kb, 128 * kb + 128)
        a64, b64 = a[:, sl].astype(np.float64), b[sl].astype(np.float64)
        s64 = sa_full[:, kb].astype(np.float64)[:, None] * sb_full[kb].astype(np.float64)[None, :]
        ex += s64 * (a64 @ b64)
        w += np.abs(s64) * (np.abs(a64) @ np.abs(b64))
    return ex, w


@gpu
@pytest.mark.parametrize("k", [1024, 4096, 16384])
def test_error_bound_on_random_operands(gemm, k):
    """Random e4m3 operands and random scales for every recipe: within rel_bound(k) of the float64 product of the
    dequantized operands (fp32 C)."""
    rng = np.random.default_rng(k)
    m, n = 160, 272
    a8 = encode(rng.standard_normal((m, k)) * 8, E4M3)
    bt8 = encode(rng.standard_normal((n, k)) * 8, E4M3)
    a, b = decode(a8, E4M3), decode(bt8, E4M3).T
    for blocks in RECIPES:
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        sa_full, sb_full = expand_scales(sa, sb, blocks, m, n)
        got = run(gemm, a8, bt8, E4M3, E4M3, dev(sa), dev(sb), blocks, None, OUT_F32).astype(np.float64)
        ex, w = exact_and_weight(a, b, sa_full, sb_full)
        err = np.abs(got - ex)
        assert bool((err <= rel_bound(k) * w).all()), (blocks, float((err / w).max()))
        print(f"k={k} {RECIPE_NAME[blocks]}: max |err| / w = {(err / w).max():.3g} (bound {rel_bound(k):.3g})")


@gpu
def test_layouts_and_pitches_match_nt(gemm):
    """NN, TN and TT, unaligned pitches and unaligned bases are bit-identical to the aligned (N, T) call."""
    rng = np.random.default_rng(31)
    m, n, k = 190, 250, 333
    ta, tb = E4M3, E5M2
    a8 = encode(rng.standard_normal((m, k)), ta)
    b8 = encode(rng.standard_normal((k, n)), tb)
    bias = round_out(rng.standard_normal(n).astype(np.float32), OUT_BF16)
    for blocks in RECIPES:
        Sa, Sb = (dev(s) for s in recipe_scales(rng, blocks, m, n, k))
        ref = run(gemm, a8, np.ascontiguousarray(b8.T), ta, tb, Sa, Sb, blocks, bias, OUT_BF16)
        for op_a in (OP_N, OP_T):
            for op_b in (OP_N, OP_T):
                sa8 = np.ascontiguousarray(a8.T) if op_a else a8
                sb8 = np.ascontiguousarray(b8.T) if op_b else b8
                got = run(gemm, sa8, sb8, ta, tb, Sa, Sb, blocks, bias, OUT_BF16, op_a, op_b)
                assert same_bits(got, ref), (blocks, op_a, op_b)
        for pad, off in ((3, 0), (0, 1), (5, 1)):
            A = np.zeros((m, k + pad + off), np.uint8)
            A[:, off:off + k] = a8
            Bt = np.zeros((n, k + pad + off), np.uint8)
            Bt[:, off:off + k] = b8.T
            Ad, Bd = dev(A), dev(Bt)
            Bi = torch.from_numpy(bias).to(torch.bfloat16).cuda()
            Cm = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            rc = gemm.lib.b200_gemm_fp8_blockwise(OP_N, OP_T, ta, tb, m, n, k, Ad.data_ptr() + off, k + pad + off,
                                                  Bd.data_ptr() + off, k + pad + off, Sa.data_ptr(), blocks[0],
                                                  *strides_of(Sa), Sb.data_ptr(), blocks[1], *strides_of(Sb),
                                                  Bi.data_ptr(), Cm.data_ptr(), n, OUT_BF16, None)
            assert rc == 0
            assert same_bits(Cm.float().cpu().numpy(), ref), (blocks, pad, off)


def scale_views(vals):
    """The same (r, c) values as CUDA tensors in four layouts: row-major, outer-dim-major (column-major), row-major
    with a padded row stride, and column-major with a padded column stride."""
    r, c = vals.shape
    v = dev(vals)
    row_pad = torch.full((r, c + 5), float("nan"), device="cuda")[:, :c]
    row_pad.copy_(v)
    col_pad = torch.full((c, r + 7), float("nan"), device="cuda")[:, :r].t()
    col_pad.copy_(v)
    return [v, v.t().contiguous().t(), row_pad, col_pad]


@gpu
def test_scale_layouts_are_bit_identical(gemm):
    """Outer-dim-major, row-major and padded k-block strides give identical bits; so does stride 0 against a
    materialised copy of the broadcast values."""
    rng = np.random.default_rng(41)
    m, n, k = 200, 300, 401
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    bt8 = np.ascontiguousarray(b8.T)
    for blocks in RECIPES:
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        ref = run(gemm, a8, bt8, E4M3, E4M3, dev(sa), dev(sb), blocks, None, OUT_F32)
        for Sa in scale_views(sa):
            for Sb in scale_views(sb):
                got = run(gemm, a8, bt8, E4M3, E4M3, Sa, Sb, blocks, None, OUT_F32)
                assert same_bits(got, ref), (blocks, Sa.stride(), Sb.stride())
        # stride 0: scale_a constant along K, scale_b constant along its columns (and along K)
        row_a = sa[:, :1]
        col_b = sb[:1, :1]
        Sa0 = dev(row_a).expand(sa.shape)
        Sb0 = dev(col_b).expand(sb.shape)
        assert Sa0.stride(1) == 0 and Sb0.stride() == (0, 0)
        want = run(gemm, a8, bt8, E4M3, E4M3, dev(np.broadcast_to(row_a, sa.shape)),
                   dev(np.broadcast_to(col_b, sb.shape)), blocks, None, OUT_F32)
        assert same_bits(run(gemm, a8, bt8, E4M3, E4M3, Sa0, Sb0, blocks, None, OUT_F32), want), blocks


def nan_fenced(vals):
    """vals as a view into a NaN-filled buffer: NaN on every side, in the same rows and columns included."""
    r, c = vals.shape
    buf = torch.full((r + 2, c + 2), float("nan"), device="cuda")
    view = buf[1:r + 1, 1:c + 1]
    view.copy_(dev(vals))
    return view


@gpu
def test_no_reads_outside_the_scales(gemm):
    """Scales fenced by NaN, with m, n and k off the 128 grid: no NaN reaches C, and C equals the oracle."""
    rng = np.random.default_rng(51)
    for m, n, k in ((200, 300, 401), (129, 131, 130), (70, 50, 60)):
        a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
        a, b = decode(a8, E4M3), decode(b8, E4M3)
        for blocks in RECIPES:
            sa, sb = recipe_scales(rng, blocks, m, n, k)
            got = run(gemm, a8, np.ascontiguousarray(b8.T), E4M3, E4M3, nan_fenced(sa), nan_fenced(sb), blocks, None,
                      OUT_F32)
            assert not np.isnan(got).any(), (m, n, k, blocks)
            assert same_bits(got, oracle_blockwise(a, b, *expand_scales(sa, sb, blocks, m, n), None, OUT_F32))


@gpu
def test_non_finite_scales(gemm):
    """A NaN in one block scale poisons exactly the rows / columns of its block; an inf scale meeting an all-zero
    block accumulator gives NaN (0 * inf); the rest equals the oracle."""
    rng = np.random.default_rng(61)
    m, n, k = 300, 400, 3 * 128 + 5
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    a8[7, 128:256] = 0                                    # row 7 of block 1 is all zero
    a, b = decode(a8, E4M3), decode(b8, E4M3)
    bt8 = np.ascontiguousarray(b8.T)
    for blocks in RECIPES:
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        if blocks[1] == 128:
            sb[2, 1] = np.nan                             # block 2 of columns [128, 256)
            nan_cols = np.arange(128, 256)
        else:
            sb[2, 33] = np.nan
            nan_cols = np.array([33])
        if blocks[0] == 1:
            sa[5, 0] = np.nan
            sa[7, 1] = np.inf
            nan_rows = np.array([5, 7])
        else:
            sa[1, 3] = np.nan                             # rows [128, 256), last k-block
            nan_rows = np.arange(128, 256)
        got = run(gemm, a8, bt8, E4M3, E4M3, dev(sa), dev(sb), blocks, None, OUT_F32)
        want_nan = np.zeros((m, n), bool)
        want_nan[nan_rows] = True
        want_nan[:, nan_cols] = True
        assert np.array_equal(np.isnan(got), want_nan), blocks
        assert same_bits_or_nan(got, oracle_blockwise(a, b, *expand_scales(sa, sb, blocks, m, n), None, OUT_F32))


@gpu
def test_fp16_output_overflows_to_inf(gemm):
    rng = np.random.default_rng(71)
    m, n, k = 130, 140, 300
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    a, b = decode(a8, E4M3), decode(b8, E4M3)
    for blocks in RECIPES:
        sa, sb = recipe_scales(rng, blocks, m, n, k, lambda r, s: (r.uniform(1, 2, s) * 64).astype(np.float32))
        got = run(gemm, a8, np.ascontiguousarray(b8.T), E4M3, E4M3, dev(sa), dev(sb), blocks, None, OUT_F16)
        assert np.isposinf(got).any() and np.isneginf(got).any()
        assert same_bits(got, oracle_blockwise(a, b, *expand_scales(sa, sb, blocks, m, n), None, OUT_F16))


@gpu
@pytest.mark.parametrize("o", [OUT_F32, OUT_BF16, OUT_F16], ids=lambda o: OUT_NAME[o])
def test_k_zero_and_empty(gemm, o):
    """k == 0 stores round_out(+0 + bias_j), or +0, and reads no scale; m == 0 or n == 0 writes nothing."""
    m, n = 70, 50
    one = torch.ones((1, 1), device="cuda")
    for with_bias in (False, True):
        bias = np.linspace(-3, 3, n).astype(np.float32)
        bias[0] = -0.0
        bias = round_out(bias, o)
        Bi = torch.from_numpy(bias).to(out_dtype(o)).cuda() if with_bias else None
        Cm = torch.full((m, n), float("nan"), dtype=out_dtype(o), device="cuda")
        rc = gemm.lib.b200_gemm_fp8_blockwise(OP_N, OP_T, E4M3, E4M3, m, n, 0, None, 0, None, 0, one.data_ptr(), 1, 0, 0,
                                              one.data_ptr(), 128, 0, 0, Bi.data_ptr() if with_bias else None,
                                              Cm.data_ptr(), n, o, None)
        assert rc == 0
        got = Cm.float().cpu().numpy()
        want = np.broadcast_to((np.float32(0) + bias) if with_bias else np.float32(0), (m, n))
        assert same_bits(np.ascontiguousarray(got), np.ascontiguousarray(want).astype(np.float32))
    for mm, nn in ((0, n), (m, 0)):
        Cm = torch.full((m, n), 7.0, dtype=out_dtype(o), device="cuda")
        rc = gemm.lib.b200_gemm_fp8_blockwise(OP_N, OP_T, E4M3, E4M3, mm, nn, 16, None, 16, None, 16, None, 1, 0, 0, None,
                                              128, 0, 0, None, Cm.data_ptr(), n, o, None)
        assert rc == 0
        assert bool((Cm == 7).all())


@gpu
def test_scaled_mm_blockwise_end_to_end(gemm):
    """scaled_mm with each recipe (torch's outer-dim-major scale_a) equals the ABI call; k <= 128 with rowwise-shaped
    scales stays on the rowwise kernel."""
    rng = np.random.default_rng(81)
    m, n, k = 200, 300, 401
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    bt8 = np.ascontiguousarray(b8.T)
    A = dev(a8).view(torch.float8_e4m3fn)
    W = dev(bt8).view(torch.float8_e4m3fn)
    for blocks in RECIPES:
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        Sa = dev(np.ascontiguousarray(sa.T)).t()                   # torch's layout: outer-dim-major
        Sb = dev(sb)
        got = gemm.scaled_mm(A, W.t(), Sa, Sb, out_dtype=torch.bfloat16)
        assert gemm.last_kernel() == "tc_e4m3_obf16_blk_128x128"
        want = run(gemm, a8, bt8, E4M3, E4M3, Sa, Sb, blocks, None, OUT_BF16)
        assert same_bits(got.float().cpu().numpy(), want), blocks
    A = dev(a8[:, :100]).view(torch.float8_e4m3fn)
    W = dev(np.ascontiguousarray(bt8[:, :100])).view(torch.float8_e4m3fn)
    gemm.scaled_mm(A, W.t(), torch.ones((m, 1), device="cuda"), torch.ones((1, 1), device="cuda"))
    assert gemm.last_kernel() == "tc_e4m3_obf16_acc_128x128"
    gemm.scaled_mm(A, W.t(), torch.ones((m, 1), device="cuda"), torch.ones((1, 3), device="cuda"))
    assert gemm.last_kernel() == "tc_e4m3_obf16_blk_128x128"


@gpu
def test_cuda_graph_with_rewritten_scales(gemm):
    """One capture, replayed with the block scales rewritten in place between replays: the host never reads them."""
    rng = np.random.default_rng(91)
    m, n, k = 256, 384, 3 * 128 + 64
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    a, b = decode(a8, E4M3), decode(b8, E4M3)
    A = dev(a8).view(torch.float8_e4m3fn)
    W = dev(np.ascontiguousarray(b8.T)).view(torch.float8_e4m3fn)
    blocks = (1, 128)
    sa0, sb0 = recipe_scales(rng, blocks, m, n, k)
    Sa, Sb = dev(sa0), dev(sb0)
    out = torch.empty((m, n), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gemm.scaled_mm(A, W.t(), Sa, Sb, out=out, stream=s)         # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gemm.scaled_mm(A, W.t(), Sa, Sb, out=out)
    for r in range(3):
        sa, sb = recipe_scales(rng, blocks, m, n, k)
        Sa.copy_(torch.from_numpy(sa))
        Sb.copy_(torch.from_numpy(sb))
        g.replay()
        torch.cuda.synchronize()
        want = oracle_blockwise(a, b, *expand_scales(sa, sb, blocks, m, n), None, OUT_F32)
        assert same_bits(out.cpu().numpy(), want), r


@gpu
def test_deepseek_v3_sized_call(gemm):
    """m = 2048, n = 7168, k = 2048, e4m3, (1 x 128, 128 x 128), bf16 out, quantised as DeepSeek-V3 does (amax / 448
    per 1 x 128 group of x and per 128 x 128 block of W): a row sample inside rel_bound(k) plus one bf16 rounding."""
    torch.manual_seed(0)
    m, n, k = 2048, 7168, 2048
    q = k // 128
    x = torch.randn(m, k, device="cuda")
    Wf = torch.randn(n, k, device="cuda") * 0.02
    sx = (x.view(m, q, 128).abs().amax(dim=2) / 448).clamp_min(1e-12)              # (m, q)
    sw = (Wf.view(n // 128, 128, q, 128).abs().amax(dim=(1, 3)) / 448).clamp_min(1e-12)   # (n / 128, q)
    xq = (x.view(m, q, 128) / sx[:, :, None]).view(m, k).to(torch.float8_e4m3fn)
    wq = (Wf.view(n // 128, 128, q, 128) / sw[:, None, :, None]).view(n, k).to(torch.float8_e4m3fn)
    scale_a = sx.t().contiguous().t()                                              # outer-dim-major, as torch takes it
    scale_b = sw.t()                                                               # (q, n / 128)
    got = gemm.scaled_mm(xq, wq.t(), scale_a, scale_b, out_dtype=torch.bfloat16)
    assert gemm.last_kernel() == "tc_e4m3_obf16_blk_128x128"
    rows = torch.arange(0, m, 97, device="cuda")
    a = xq[rows].float().cpu().numpy()
    b = wq.float().cpu().numpy().T
    sa_full = sx[rows].cpu().numpy()
    sb_full = np.repeat(sw.t().cpu().numpy(), 128, axis=1)
    ex, w = exact_and_weight(a, b, sa_full, sb_full)
    err = np.abs(got[rows].double().cpu().numpy() - ex)
    assert bool((err <= rel_bound(k) * w + 2.0 ** -8 * np.abs(ex)).all())


@gpu
def test_against_torch_scaled_mm(gemm):
    """torch._scaled_mm with blockwise scales: compared where torch accepts them, else skipped with its refusal."""
    torch.manual_seed(1)
    m, n, k = 256, 512, 1024
    q = k // 128
    xq = (torch.randn(m, k, device="cuda") * 8).to(torch.float8_e4m3fn)
    wq = (torch.randn(n, k, device="cuda") * 8).to(torch.float8_e4m3fn)
    sa = (torch.rand(q, m, device="cuda") + 0.5).t()                               # (m, q), outer-dim-major
    sb = (torch.rand(n // 128, q, device="cuda") + 0.5).t()                        # (q, n / 128)
    try:
        want = torch._scaled_mm(xq, wq.t(), sa, sb, out_dtype=torch.float32)
    except (RuntimeError, NotImplementedError, ValueError) as e:
        pytest.skip(f"torch._scaled_mm refuses blockwise scales: {str(e).splitlines()[0]}")
    got = gemm.scaled_mm(xq, wq.t(), sa, sb, out_dtype=torch.float32)
    a, b = xq.float().cpu().numpy(), wq.float().cpu().numpy().T
    ex, w = exact_and_weight(a, b, sa.cpu().numpy(), np.repeat(sb.cpu().numpy(), 128, axis=1))
    assert bool((np.abs(got.double().cpu().numpy() - ex) <= rel_bound(k) * w).all())
    assert bool((np.abs(want.double().cpu().numpy() - got.double().cpu().numpy()) <= 2 * rel_bound(k) * w).all())
