"""Each fp32 mode of b200_gemm_f32 against an exact model of its arithmetic, over the whole fp32 range.

The models (tests/_fp32_model.py) restate the operand transform of TF32, BF16X3, BF16X2 and F16X2 and sum the
plane products the kernel issues in float64.  Three kinds of GPU check use them:

  known answers   dyadic operands whose plane products are all multiples of one quantum q per output element,
                  with the sum of their absolute values below 2^24 q: fp32 accumulation in any order (chopping
                  tensor-core adds, chunk folds, K-split folds) is then exact, so the GPU must equal the model
                  bit for bit, through every route that forms split planes.  The CPU tests below check those two
                  conditions and show that a wrong product list, a wrong rounding of the split or a wrong F16X2
                  exponent changes the expected bits.
  random          uniform and wide-range (2^+-60 within a row / column) operands: |GPU - model| within a bound
                  from the fp32 accumulation alone, and |model - exact| within the mode's documented class.
  full range      rows of A and columns of B from 2^-149 to FLT_MAX, inf and NaN: STRICT (and the generic kernel)
                  bit-exact against the oracle, non-finite results exactly where the IEEE result is non-finite in
                  every mode, finite results within the mode's class.

A chopped (instead of rounded) split changes BF16X3 and F16X2 only through the products they drop, by less than
2^-23 of |a||b|: no test can tell it apart, and it would not change their error class.  BF16X2 runs the same
split kernel as BF16X3 (split_planes_kernel<NP>) and shows the rounding.

The library's debug hooks are process-global: the `hooks` fixture restores them after every test."""
import numpy as np
import pytest

import _fp32_model as fm
import _libs

try:
    import torch
except ImportError:          # the model tests need no torch
    torch = None

gpu = pytest.mark.gpu
F32_MAX = fm.F32_MAX
SPLIT_MODES = ("bf16x3", "bf16x2", "f16x2")
TC_MODES = ("tf32",) + SPLIT_MODES
KERNEL = {"tf32": "tc_tf32_128x128", "bf16x3": "tc_bf16x3_128x128", "bf16x2": "tc_bf16x2_128x128",
          "f16x2": "tc_f16x2_128x128"}
CHUNK = {"tf32": 0, "bf16x3": 512, "bf16x2": 512, "f16x2": 1024}     # built-in accumulation chunks (K)


def f32(x):
    return np.asarray(x, np.float32)


# ==== worked examples of the model (no GPU) ===============================================================
def test_bf16_planes_worked_examples():
    one = 1 + 2.0 ** -9 + 2.0 ** -18
    p = fm.bf16_planes(f32([one]), 3)
    assert [float(x[0]) for x in p] == [1.0, 2.0 ** -9, 2.0 ** -18]
    # FLT_MAX: the first plane would round to inf; it is clamped to 0x7f7f and the residual stays exact
    p = fm.bf16_planes(f32([F32_MAX]), 3)
    assert fm.bits(p[0])[0] == 0x7F7F0000
    assert sum(float(x[0]) for x in p) == F32_MAX
    big = fm.from_bits([0x7F7F8000])               # the smallest finite value RNE sends to bf16 inf
    p = fm.bf16_planes(big, 3)
    assert fm.bits(p[0])[0] == 0x7F7F0000 and float(p[1][0]) == 2.0 ** 119 and float(p[2][0]) == 0.0
    assert fm.bits(fm.bf16_round(big))[0] == 0x7F800000
    p = fm.bf16_planes(-big, 2)
    assert fm.bits(p[0])[0] == 0xFF7F0000 and float(p[1][0]) == -(2.0 ** 119)
    tiny = fm.from_bits([1])                       # 2^-149: below the bf16 subnormal quantum 2^-133
    p = fm.bf16_planes(tiny, 3)
    assert [float(x[0]) for x in p] == [0.0, 0.0, 0.0]
    p = fm.bf16_planes(f32([2.0 ** -133 + 2.0 ** -149]), 3)      # bf16 subnormal plane, the rest is lost
    assert [float(x[0]) for x in p] == [2.0 ** -133, 0.0, 0.0]
    for v in (np.inf, -np.inf):                    # non-finite: p1 = x, lower planes zero (not NaN)
        p = fm.bf16_planes(f32([v]), 3)
        assert float(p[0][0]) == v and float(p[1][0]) == 0.0 and float(p[2][0]) == 0.0
    p = fm.bf16_planes(f32([np.nan]), 3)
    assert np.isnan(p[0][0]) and float(p[1][0]) == 0.0
    # ties go to even; chopping differs
    x = f32([1 + 2.0 ** -9 - 2.0 ** -18])
    assert [float(v[0]) for v in fm.bf16_planes(x, 3)] == [1.0, 2.0 ** -9, -(2.0 ** -18)]
    assert [float(v[0]) for v in fm.bf16_planes(x, 3, trunc=True)] == [1.0, 2.0 ** -9 - 2.0 ** -17, 2.0 ** -18]


def test_pow2_exp_worked_examples():
    vals = f32([0.0, fm.from_bits([1])[0], 2.0 ** -127, 2.0 ** -126, 1.0, 2.0 ** 127, F32_MAX, np.inf, np.nan,
                0.75, fm.from_bits([0x007FFFFF])[0]])
    want = [0, -148, -126, -125, 1, 128, 128, 0, 0, 0, -126]
    assert fm.pow2_exp(vals).tolist() == want
    for v, e in zip(vals, want):                   # maxv * 2^-e in [0.5, 1) for finite nonzero maxima
        if np.isfinite(v) and v != 0:
            assert 0.5 <= float(v) * 2.0 ** -e < 1.0


def test_f16_and_tf32_worked_examples():
    # F16X2 planes of a subnormal-maximum row: scaled by 2^148, nothing is lost
    row = f32([[fm.from_bits([3])[0], fm.from_bits([1])[0]]])
    e = fm.pow2_exp(fm.absmax(row, 1))
    assert e.tolist() == [-147]
    h1, h2 = fm.f16_planes(row, e[:, None])
    assert (h1 + h2).tolist() == [[0.75, 0.25]]
    # h2 keeps fp16 subnormals: x' = 0.5 + 2^-24 -> h1 = 0.5, h2 = 2^-24
    h1, h2 = fm.f16_planes(f32([[0.5 + 2.0 ** -24]]), np.zeros((1, 1), np.int64))
    assert float(h1[0, 0]) == 0.5 and float(h2[0, 0]) == 2.0 ** -24
    # tf32 drops 13 bits (chops); a finite value stays finite, inf / NaN stay
    x = f32([1 + 2.0 ** -10 + 2.0 ** -11 + 2.0 ** -12, F32_MAX, np.inf, -np.inf])
    t = fm.tf32(x)
    assert float(t[0]) == 1 + 2.0 ** -10 and float(t[1]) == float(fm.from_bits([0x7F7FE000])[0])
    assert np.isinf(t[2]) and np.isinf(t[3])
    assert float(fm.tf32(x, rne=True)[0]) == 1 + 2.0 ** -9


def test_model_equals_exact_product_for_exact_planes():
    """Operands whose planes hold every bit: BF16X3 of 24-bit values misses only the dropped products."""
    rng = np.random.default_rng(1)
    A, B = f32(rng.uniform(-1, 1, (16, 64))), f32(rng.uniform(-1, 1, (64, 12)))
    exact = A.astype(np.float64) @ B.astype(np.float64)
    for mode in TC_MODES:
        err = np.abs(fm.model(A, B, mode) - exact)
        assert (err <= fm.class_bound(A, B, mode)).all(), mode
    # BF16X3 with all nine products is exact
    nine = tuple((i, j) for i in range(3) for j in range(3))
    assert np.abs(fm.model(A, B, "bf16x3", prods=nine) - exact).max() <= 1e-15 * np.abs(exact).max()


# ==== known-answer operands ===============================================================================
def ka_operands(mode, m, n, k, seed):
    """Dyadic A (m x k), B (k x n) with known planes.  Entries are sparse so that few products meet per output.

    bf16x3 / bf16x2: +-(1 + s2 2^-9 + s3 2^-18) 2^E, (s2, s3) in {(1, 1), (1, 0), (1, -1), (-1, 1), (-1, 0),
    (0, 0)} (planes +-2^E, +-2^(E-9), +-2^(E-18); ties to even included.  1 - 2^-9 - 2^-18 would round to
    1 - 2^-8, and s2 = 0 would move 2^-18 into the second plane: either spreads the bits of the products).
    f16x2: x' = h1 + h2, h1 in {+-0.5, +-0.75}, h2 in {0, +-2^-13, +-2^-14}, times 2^e of the row / column.
    tf32: +-{1, 1.125, 1.5, 1.75} 2^E plus 3 2^(E-12), which tf32 chops away (rounding would not).
    E per row of A / column of B in [-2, 2]."""
    rng = np.random.default_rng(seed)
    dens = min(1.0, (16.0 / k) ** 0.5)

    def make(r, c, axis):
        sign = rng.choice([-1.0, 1.0], (r, c))
        scale = np.ldexp(1.0, rng.integers(-2, 3, r if axis == 1 else c))
        scale = scale[:, None] if axis == 1 else scale[None, :]
        if mode in ("bf16x3", "bf16x2"):
            s = np.array([(1, 1), (1, 0), (1, -1), (-1, 1), (-1, 0), (0, 0)])[rng.integers(0, 6, (r, c))]
            v = 1 + s[..., 0] * 2.0 ** -9 + s[..., 1] * 2.0 ** -18
        elif mode == "f16x2":
            v = rng.choice([0.5, 0.75], (r, c)) + rng.choice([0, 2.0 ** -13, -2.0 ** -13, 2.0 ** -14, -2.0 ** -14], (r, c))
        else:
            v = rng.choice([1.0, 1.125, 1.5, 1.75], (r, c)) + rng.choice([0, 3 * 2.0 ** -12], (r, c))
        x = sign * v * scale * (rng.random((r, c)) < dens)
        out = f32(x)
        assert (out.astype(np.float64) == x).all()
        return out
    return make(m, k, 1), make(k, n, 0)


def lowbit(x):
    """Least significant set bit of each nonzero dyadic float64 (inf where x == 0)."""
    x = np.abs(np.asarray(x, np.float64))
    mant, ex = np.frexp(x)
    mi = (mant * 2.0 ** 53).astype(np.int64)
    tz = np.zeros_like(mi)
    for s in (32, 16, 8, 4, 2, 1):
        low = (mi & ((1 << s) - 1)) == 0
        low &= mi != 0
        tz = np.where(low, tz + s, tz)
        mi = np.where(low, mi >> s, mi)
    return np.where(x == 0, np.inf, np.ldexp(1.0, (ex - 53 + tz).astype(np.int64)))


def exact_accumulation_margin(A, B, mode, alpha=1.0, c0=None, beta=0.0):
    """Per output element, 2^24 q / (sum of |terms|): > 1 means every fp32 partial sum is exact in any order.
    q is the smallest lowbit of any plane product meeting at (i, j) (in the accumulator's units), and also of
    alpha * q and of beta * C0."""
    pa, pb, ea, eb = fm.planes(A, B, mode)
    q = np.full((A.shape[0], B.shape[1]), np.inf)
    for i, j in fm.PRODS[mode]:
        q = np.minimum(q, lowbit(pa[i]).min(1)[:, None] * lowbit(pb[j]).min(0)[None, :])
    S = fm.model(A, B, mode, absolute=True)
    if mode == "f16x2":               # the accumulator sums scaled products; the unscale is exact
        unit = np.ldexp(1.0, (ea[:, None] + eb[None, :]).astype(np.int64))
        q = q * unit
    q = q * min(alpha, 1.0)
    total = alpha * S
    if c0 is not None and beta != 0.0:
        bc = np.abs(beta * c0.astype(np.float64))
        q = np.minimum(q, lowbit(bc))                 # beta * C0 is one more term of the sum
        total = total + bc
    q = np.where(np.isinf(q), 1.0, q)
    return 2.0 ** 24 * q / np.maximum(total, 1e-300)


KA_SHAPES = {"plain": (200, 136, 160), "chunk64": (200, 136, 200), "split_tail": (128, 128, 520)}


def ka_case(mode, route, seed=0):
    m, n, k = KA_SHAPES.get(route, KA_SHAPES["plain"])
    A, B = ka_operands(mode, m, n, k, 1000 + seed + 17 * TC_MODES.index(mode))
    c0 = f32(np.random.default_rng(seed).integers(-64, 65, (m, n)) * 2.0 ** -10)
    return A, B, c0


KA_ALPHA, KA_BETA = 2.0, -0.5


def ka_expected(A, B, c0, mode, route):
    want = fm.model(A, B, mode)
    if route == "acc":
        want = want + c0
    elif route == "ex":
        want = KA_ALPHA * want + KA_BETA * c0.astype(np.float64)
    return want


@pytest.mark.parametrize("mode", TC_MODES)
def test_known_answer_operands_are_exact(mode):
    """The two conditions under which any fp32 accumulation order reproduces the model exactly."""
    for route in ("plain", "chunk64", "split_tail"):
        A, B, c0 = ka_case(mode, route)
        margin = exact_accumulation_margin(A, B, mode)
        assert margin.min() > 1.0, (route, margin.min())
        want = ka_expected(A, B, c0, mode, route)
        assert (f32(want).astype(np.float64) == want).all()
        assert np.count_nonzero(want) > want.size // 2
    A, B, c0 = ka_case(mode, "plain")
    for alpha, beta in ((1.0, 1.0), (KA_ALPHA, KA_BETA)):
        margin = exact_accumulation_margin(A, B, mode, alpha, c0, beta)
        assert margin.min() > 1.0, (alpha, beta)


def mutants(mode):
    P = fm.PRODS[mode]
    out = []
    for i in range(len(P)):
        out.append((f"drop{P[i]}", dict(prods=P[:i] + P[i + 1:])))
        out.append((f"dup{P[i]}", dict(prods=P + (P[i],))))
    if mode in ("bf16x2", "tf32"):
        out.append(("chopped split" if mode == "bf16x2" else "rounded tf32", dict(trunc=True)))
    if mode == "f16x2":
        out += [("h2 dropped", dict(drop_h2=True)), ("scale exponent +1", dict(exp_shift=1)),
                ("scale exponent -1", dict(exp_shift=-1)), ("unscale exponent +1", dict(unscale_shift=1))]
    return out


@pytest.mark.parametrize("mode", TC_MODES)
def test_mutants_change_expected_bits(mode):
    """Every mutant of the model gives other fp32 bits than the model for the known-answer operands of every
    route, so the bit-exact GPU tests would catch such a kernel."""
    for route in ("plain", "chunk64", "split_tail"):
        A, B, _ = ka_case(mode, route)
        want = fm.bits(f32(fm.model(A, B, mode)))
        for name, kw in mutants(mode):
            got = fm.bits(f32(fm.model(A, B, mode, **kw)))
            assert not np.array_equal(got, want), (route, name)


# ==== GPU helpers ===========================================================================================
@pytest.fixture
def hooks(gemm):
    """The library's debug hooks, reset to their defaults after the test whatever its outcome."""
    lib = gemm.lib
    try:
        yield lib
    finally:
        lib.b200_gemm_debug_set_bn(0)
        lib.b200_gemm_debug_set_split_tail(1)
        lib.b200_gemm_debug_set_group_rows(0)
        lib.b200_gemm_debug_set_ffma_variant(-1)
        lib.b200_gemm_debug_set_split_chunk(-1, -1)


def mode_id(gemm, mode):
    return {"strict": gemm.F32_STRICT, "tf32": gemm.F32_TF32, "bf16x3": gemm.F32_BF16X3, "bf16x2": gemm.F32_BF16X2,
            "f16x2": gemm.F32_F16X2, "auto": gemm.F32_AUTO}[mode]


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def nan_out(m, n):
    """(buffer with an odd pitch, m x n view), NaN filled."""
    buf = torch.full((m, n + 1 + n % 2), float("nan"), device="cuda")
    return buf, buf[:, :n]


# ==== known answers, bit-exact ===============================================================================
KA_ROUTES = {"tf32": ("plain", "acc", "ex", "split_tail"),
             "bf16x3": ("plain", "acc", "ex", "packed_b", "chunk64", "split_tail"),
             "bf16x2": ("plain", "acc", "ex", "packed_b", "chunk64", "split_tail"),
             "f16x2": ("plain", "acc", "ex", "packed_b", "packed_ab", "chunk64", "split_tail")}


@gpu
@pytest.mark.parametrize("mode,route", [(md, r) for md in TC_MODES for r in KA_ROUTES[md]])
def test_known_answer_bit_exact(gemm, hooks, mode, route):
    """Dyadic operands (exact accumulation in any order): every route equals the model bit for bit."""
    A, B, c0 = ka_case(mode, route)
    m, n = A.shape[0], B.shape[1]
    margin = exact_accumulation_margin(A, B, mode, KA_ALPHA if route == "ex" else 1.0, c0, KA_BETA)
    assert margin.min() > 1.0
    Ad, Bd = dev(A), dev(B)
    buf, out = nan_out(m, n)
    md = mode_id(gemm, mode)
    if route in ("acc", "ex"):
        out.copy_(dev(c0))
    if route == "chunk64":
        hooks.b200_gemm_debug_set_split_chunk(64, 64)
    if route in ("plain", "chunk64", "split_tail"):
        gemm.gemm_f32(Ad, Bd, out=out, mode=md)
    elif route == "acc":
        gemm.gemm_f32(Ad, Bd, out=out, mode=md, accumulate=True)
    elif route == "ex":
        gemm.gemm_f32_ex(KA_ALPHA, Ad, Bd, KA_BETA, out, mode=md)
    elif route == "packed_b":
        pb = gemm.PackedB(Bd, md)
        gemm.gemm_f32_packed(Ad, pb, out=out)
        pb.close()
    elif route == "packed_ab":                       # two K-slices of B against column ranges of one packed A
        k1 = 80
        pa = gemm.PackedA(Ad, md)
        pbs = [gemm.PackedB(Bd[:k1].contiguous(), md), gemm.PackedB(Bd[k1:].contiguous(), md)]
        gemm.gemm_f32_packed_ab(pa, pbs[0], out, a_k0=0)
        gemm.gemm_f32_packed_ab(pa, pbs[1], out, a_k0=k1, accumulate=True)
        for p in pbs + [pa]:
            p.close()
    assert gemm.last_kernel() == KERNEL[mode]
    got = out.cpu().numpy()
    want = f32(ka_expected(A, B, c0, mode, route))
    bad = fm.bits(got) != fm.bits(want)
    assert not bad.any(), (int(bad.sum()), got[bad][:4], want[bad][:4])
    assert bool(torch.isnan(buf[:, n:]).all())


# ==== random and wide-range operands ===========================================================================
def random_operands(kind, m, n, k, seed):
    rng = np.random.default_rng(seed)
    A, B = rng.uniform(-1, 1, (m, k)), rng.uniform(-1, 1, (k, n))
    if kind == "wide":                   # exponents spread by 2^+-60 within each row of A and column of B
        A = A * np.ldexp(1.0, rng.integers(-60, 61, (m, k)))
        B = B * np.ldexp(1.0, rng.integers(-60, 61, (k, n)))
    return f32(A), f32(B)


@gpu
@pytest.mark.parametrize("kind", ["uniform", "wide"])
@pytest.mark.parametrize("mode", TC_MODES)
def test_random_against_model(gemm, hooks, mode, kind):
    """GPU vs its own model within the fp32 accumulation bound (this catches wrong arithmetic), and the model vs
    the exact product within the mode's documented class.  256 x 256 x 1024 has a 4-way K-split tail."""
    m, n, k = 256, 256, 1024
    A, B = random_operands(kind, m, n, k, 7 + TC_MODES.index(mode))
    out = gemm.gemm_f32(dev(A), dev(B), mode=mode_id(gemm, mode))
    assert gemm.last_kernel() == KERNEL[mode]
    got = out.cpu().numpy().astype(np.float64)
    mod = fm.model(A, B, mode)
    bound = fm.accumulation_bound(A, B, mode, CHUNK[mode], parts=4)
    err = np.abs(got - mod)
    assert (err <= bound).all(), float((err / bound).max())
    exact = A.astype(np.float64) @ B.astype(np.float64)
    cls = np.abs(mod - exact) / fm.class_bound(A, B, mode)
    assert (cls <= 1).all(), float(cls.max())


# ==== full-range contract ======================================================================================
def range_operands(m, n, k, seed):
    """A (m x k), B (k x n) over the whole fp32 range.  Rows of A and columns of B are scaled by 2^e with e cycling
    over -149 ... 127 (all-subnormal rows / columns at the low end); one row of A holds FLT_MAX and 0x7f7f8000
    (the rest near 2^127); a row [2^127, 1e-30, 0...] and a column [1e-30, 2^127, 0...]^T give a finite result
    through an F16X2 unscale of 2^256; inf, -inf and NaN sit at chosen (i, k) and (k, j)."""
    rng = np.random.default_rng(seed)
    ea = np.array([-149, -140, -130, -126, -120, -100, -80, -60, -30, 0, 20, 60, 100, 120, 126, 127])
    eb = np.array([-149, -141, -128, -120, -90, -60, -20, 0, 30, 60, 90, 110, 126, 127, -10, 5])
    A = rng.uniform(0.5, 1, (m, k)) * rng.choice([-1.0, 1.0], (m, k))
    B = rng.uniform(0.5, 1, (k, n)) * rng.choice([-1.0, 1.0], (k, n))
    A = A * np.ldexp(1.0, ea[np.arange(m) % len(ea)])[:, None]
    B = B * np.ldexp(1.0, eb[np.arange(n) % len(eb)])[None, :]
    A, B = f32(A), f32(B)
    big = 17                              # row with its maximum in [0x7f7f8000, FLT_MAX]
    A[big] = f32(np.abs(A[big]) * 0 + rng.uniform(1.0, 1.9, k) * 2.0 ** 127) * np.sign(A[big])
    A[big, 0], A[big, 3] = F32_MAX, -fm.from_bits([0x7F7F8000])[0]
    iu, ju = 33, 35                       # 2^127 x 1e-30 + 1e-30 x 2^127 (F16X2 unscale by 2^256)
    A[iu] = 0
    A[iu, 0], A[iu, 1] = 2.0 ** 127, 1e-30
    B[:, ju] = 0
    B[0, ju], B[1, ju] = 1e-30, 2.0 ** 127
    A[5, 7], A[50, 9], A[77, 100] = np.inf, -np.inf, np.nan
    B[11, 40], B[200 % k, 61], B[3, 90] = np.inf, np.nan, -np.inf
    return A, B


def ieee_expectations(A, B):
    """(exact product of the finite parts, must be non-finite, must be finite).  Non-finite: a row of A or a
    column of B holding inf or NaN, or |exact| >= 2 FLT_MAX.  Finite: neither, and sum |A||B| <= FLT_MAX / 4
    (so no rounding and no partial sum of any mode can decide finiteness)."""
    fa, fb = np.isfinite(A), np.isfinite(B)
    A64, B64 = np.where(fa, A, 0).astype(np.float64), np.where(fb, B, 0).astype(np.float64)
    exact = A64 @ B64
    absum = np.abs(A64) @ np.abs(B64)
    bad = (~fa.all(1))[:, None] | (~fb.all(0))[None, :]
    nonfinite = bad | (np.abs(exact) >= 2 * F32_MAX)
    finite = ~bad & (absum <= F32_MAX / 4)
    return exact, nonfinite, finite


RANGE_ROUTES = {
    # route: (mode, shape, kernel the library must report)
    "strict": ("strict", (256, 256, 256), "ffma_128x128x32_tma"),
    "generic_odd_lda": ("strict", (256, 256, 256), "generic_f32_64x64"),
    "tf32": ("tf32", (256, 256, 256), KERNEL["tf32"]),
    "bf16x3": ("bf16x3", (256, 256, 256), KERNEL["bf16x3"]),
    "bf16x2": ("bf16x2", (256, 256, 256), KERNEL["bf16x2"]),
    "f16x2": ("f16x2", (256, 256, 256), KERNEL["f16x2"]),
    "auto_strict": ("auto", (256, 256, 256), "ffma_128x128x32_tma"),            # m n k <= 2e8
    "auto_bf16x3": ("auto", (1024, 1024, 640), KERNEL["bf16x3"]),               # 2e8 < m n k < 1.3e9
    "auto_f16x2": ("auto", (1152, 1152, 1024), KERNEL["f16x2"]),                # m n k >= 1.3e9
}
AUTO_MODEL = {"auto_bf16x3": "bf16x3", "auto_f16x2": "f16x2"}


@gpu
@pytest.mark.parametrize("route", list(RANGE_ROUTES))
def test_full_range_contract(gemm, oracle, hooks, route):
    """(a) STRICT and the generic kernel bit-exact against the oracle's fused reference, subnormals and NaN
    positions included; (b) non-finite exactly where the IEEE result is (NaN or inf may differ in the split
    modes); (c) finite results within the mode's class, and the tensor-core modes within the accumulation bound
    of their model."""
    mode, (m, n, k), name = RANGE_ROUTES[route]
    if mode == "auto" and gemm.lib.b200_gemm_default_f32_mode() != gemm.F32_F16X2:
        pytest.skip("the default fp32 mode was changed in the environment")
    A, B = range_operands(m, n, k, 42)
    if route == "generic_odd_lda":
        buf = torch.zeros((m, k + 1), device="cuda")
        buf[:, :k] = dev(A)
        Ad = buf[:, :k]
    else:
        Ad = dev(A)
    cbuf, out = nan_out(m, n)
    gemm.gemm_f32(Ad, dev(B), out=out, mode=mode_id(gemm, mode))
    assert gemm.last_kernel() == name
    got = out.cpu().numpy()
    assert bool(torch.isnan(cbuf[:, n:]).all())
    exact, nonfinite, finite = ieee_expectations(A, B)
    assert nonfinite.sum() > 0 and finite.sum() > 0 and (np.abs(exact[finite]) < 2.0 ** -126).sum() > 0
    if mode in ("strict",) or route == "auto_strict":
        want = _libs.ref_f32_fma(oracle, A, B)
        assert np.array_equal(np.isnan(got), np.isnan(want))
        same = (fm.bits(got) == fm.bits(want)) | (np.isnan(got) & np.isnan(want))
        assert same.all(), int((~same).sum())
        return
    gm = AUTO_MODEL.get(route, mode)
    isfin = np.isfinite(got)
    assert not isfin[nonfinite].any(), int(isfin[nonfinite].sum())           # (b)
    assert isfin[finite].all(), np.argwhere(finite & ~isfin)[:5].tolist()
    with np.errstate(invalid="ignore", over="ignore"):
        mod = fm.model(A, B, gm)
        cls = fm.class_bound(A, B, gm)
        acc = fm.accumulation_bound(A, B, gm, CHUNK[gm], parts=4)
    g64 = got.astype(np.float64)
    err_model = np.abs(g64 - mod)[finite]
    assert (err_model <= acc[finite]).all(), float((err_model / acc[finite]).max())   # GPU vs its model
    err = np.abs(g64 - exact)[finite]
    assert (err <= cls[finite] + acc[finite]).all(), float((err / (cls[finite] + acc[finite])).max())   # (c)


# ==== subnormal operands and products on the tensor cores ========================================================
@gpu
def test_tensor_cores_keep_subnormals(gemm):
    """wgmma with subnormal bf16 / tf32 inputs, subnormal fp32 products, and fp16 subnormal planes (F16X2's h2):
    nothing is flushed to zero.  Every product and sum here is exact."""
    m = n = 128
    k = 64
    A = np.zeros((m, k), np.float32)
    B = np.zeros((k, n), np.float32)
    A[:, 0] = 2.0 ** -130            # bf16 / tf32 subnormal input
    B[0, 0::2] = 2.0 ** 100          # -> 2^-30 in even columns
    A[:, 1] = 2.0 ** -70
    B[1, 1::2] = 2.0 ** -70          # -> 2^-140, a subnormal product, in odd columns
    want = np.tile(f32([2.0 ** -30, 2.0 ** -140]), (m, n // 2))
    for mode in ("tf32", "bf16x3", "bf16x2"):
        got = gemm.gemm_f32(dev(A), dev(B), mode=mode_id(gemm, mode)).cpu().numpy()
        assert np.array_equal(got, want), (mode, got[0, :2])
    # F16X2: x' = 0.5 + 2^-24 has h2 = 2^-24, the smallest fp16 subnormal
    A = np.zeros((m, k), np.float32)
    B = np.zeros((k, n), np.float32)
    A[:, 0] = 0.5 + 2.0 ** -24
    B[0, :] = 0.5
    got = gemm.gemm_f32(dev(A), dev(B), mode=gemm.F32_F16X2).cpu().numpy()
    assert (got == f32(0.25 + 2.0 ** -25)).all(), got[0, 0]
