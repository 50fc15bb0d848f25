"""FP8 tensor-core GEMMs (b200_gemm_fp8) and scaled_mm(): torch._scaled_mm's contract.

    C = round_out( (acc * sa_i) * sb_j + bias_j )

acc is op(A) op(B) of the FP8 operands; each step is one fp32 round-to-nearest operation.  The oracle here decodes the
operands with torch's CPU casts and applies that op order in numpy float32.  On operands whose every partial sum is an
integer below 2^11 (and power-of-two scales) acc is exact in either accumulation mode, so every kernel, width, layout,
pitch and tail must equal the oracle bit for bit.  On random operands the promoted mode (fast_accum = 0) must stay
inside the bound derived from the tensor core's retained FP8 accumulation precision (measured below by crafted sums,
DESIGN §4.7) and an fp32 running sum over 128-element chunks.

The argument checks, the Python refusals and layout resolution, and the oracle against torch._scaled_mm on the CPU
need no GPU."""
import numpy as np
import pytest

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
OP_N, OP_T = 0, 1
E4M3, E5M2 = 0, 1
OUT_F32, OUT_BF16, OUT_F16 = 0, 1, 2
PAIRS = [(E4M3, E4M3), (E4M3, E5M2), (E5M2, E4M3)]
PAIR_NAME = {(E4M3, E4M3): "e4m3", (E4M3, E5M2): "e4m3e5m2", (E5M2, E4M3): "e5m2e4m3"}
OUT_NAME = {OUT_F32: "of32", OUT_BF16: "obf16", OUT_F16: "of16"}
# The tensor core's retained precision when it adds FP8 products into its fp32 accumulator: bits of significand kept,
# relative to the accumulator's leading bit (measured by test_retained_accumulation_precision; DESIGN §4.7).
RETAINED_BITS = 14
CHUNK = 128                  # K elements per promoted chunk


def _has_gpu():
    try:
        return torch is not None and torch.cuda.is_available()
    except Exception:
        return False


def fp8_dtype(t):
    return torch.float8_e4m3fn if t == E4M3 else torch.float8_e5m2


def out_dtype(o):
    return {OUT_F32: torch.float32, OUT_BF16: torch.bfloat16, OUT_F16: torch.float16}[o]


def decode(u8, t):
    """FP8 bytes (numpy uint8) -> float32 values, by torch's CPU cast."""
    return torch.from_numpy(np.ascontiguousarray(u8)).view(fp8_dtype(t)).float().numpy()


def encode(x, t):
    """float values -> FP8 bytes (numpy uint8), by torch's CPU cast (round to nearest)."""
    return torch.from_numpy(np.asarray(x, np.float32)).to(fp8_dtype(t)).view(torch.uint8).numpy()


def round_out(x32, o):
    """float32 -> the output type's values, by torch's CPU cast (round to nearest even), returned as float32."""
    return torch.from_numpy(np.asarray(x32, np.float32)).to(out_dtype(o)).float().numpy()


def oracle(a, b, sa, sb, bias, o, acc=None):
    """The contract on decoded operands a (m x k) and b (k x n), float32 scale vectors sa (m) and sb (n), a float32 bias
    (n) of the output's values or None.  acc: the exact product (float64, rounded to float32 here) unless given."""
    if acc is None:
        acc = a.astype(np.float64) @ b.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        x = (acc.astype(np.float32) * sa[:, None].astype(np.float32)) * sb[None, :].astype(np.float32)
        if bias is not None:
            x = x + bias[None, :].astype(np.float32)
    return round_out(x, o)


# ==== the C ABI through ctypes =====================================================================================
def call(gemm, op_a=OP_N, op_b=OP_T, ta=E4M3, tb=E4M3, m=4, n=4, k=4, a=1, lda=None, b=1, ldb=None, sa=1, sa_row=0,
         sb=1, sb_col=0, bias=None, c=1, ldc=None, out=OUT_BF16, fast=0):
    """b200_gemm_fp8 with raw pointers (ints; 1 stands for a dummy non-null pointer where no GPU is present)."""
    lda = lda if lda is not None else (m if op_a else k)
    ldb = ldb if ldb is not None else (k if op_b else n)
    ldc = ldc if ldc is not None else n
    return gemm.lib.b200_gemm_fp8(op_a, op_b, ta, tb, m, n, k, a, lda, b, ldb, sa, sa_row, sb, sb_col, bias, c, ldc, out,
                                  fast, None)


def test_fp8_argument_validation(gemm):
    """Refusals before the device is touched, each at its exact bound: they hold with or without a GPU."""
    assert call(gemm, ta=2) == -1 and call(gemm, tb=-1) == -1
    assert call(gemm, out=3) == -1 and call(gemm, out=-1) == -1
    assert call(gemm, sa_row=2) == -1 and call(gemm, sb_col=-1) == -1
    assert call(gemm, fast=2) == -1 and call(gemm, fast=-1) == -1
    assert call(gemm, op_a=2) == -1 and call(gemm, op_b=-1) == -1
    assert call(gemm, m=-1) == -1 and call(gemm, n=-1) == -1 and call(gemm, k=-1) == -1
    assert call(gemm, ta=E5M2, tb=E5M2) == -3                     # torch has no e5m2 x e5m2 either
    assert call(gemm, ta=E5M2, tb=E5M2, m=0) == -3
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            m, n, k = 5, 6, 7
            lda_min, ldb_min = (m if op_a else k), (k if op_b else n)
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, lda=lda_min - 1) == -1
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, ldb=ldb_min - 1) == -1
            assert call(gemm, op_a, op_b, m=m, n=n, k=k, ldc=n - 1) == -1
    assert call(gemm, a=None) == -1 and call(gemm, b=None) == -1 and call(gemm, c=None) == -1
    assert call(gemm, sa=None) == -1 and call(gemm, sb=None) == -1   # a null scale with work to do
    assert call(gemm, sa=None, k=0) == -1
    # m == 0 or n == 0: a no-op, null pointers included
    assert call(gemm, m=0, a=None, b=None, c=None, sa=None, sb=None) == 0
    assert call(gemm, n=0, a=None, b=None, c=None, sa=None, sb=None) == 0


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_fp8_accepts_at_the_bounds_without_device(gemm):
    """The smallest legal ld, k == 0 with null operands, and every accepted pair reach the device check (-2)."""
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            assert call(gemm, op_a, op_b, m=5, n=6, k=7) == -2
    assert call(gemm, k=0, a=None, b=None) == -2
    for ta, tb in PAIRS:
        for o in (OUT_F32, OUT_BF16, OUT_F16):
            for fast in (0, 1):
                assert call(gemm, ta=ta, tb=tb, out=o, fast=fast, sa_row=1, sb_col=1) == -2


# ==== scaled_mm: refusals and layouts (CPU) ========================================================================
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")


def _fp8(shape, t=E4M3, device="cpu"):
    return torch.zeros(shape, dtype=torch.float32, device=device).to(fp8_dtype(t))


@need_torch
def test_scaled_mm_refusals(gemm):
    A, B = _fp8((8, 16)), _fp8((16, 4))
    one = torch.ones(1)
    with pytest.raises(TypeError):
        gemm.scaled_mm(_fp8((8, 16), E5M2), _fp8((16, 4), E5M2), one, one)
    with pytest.raises(TypeError):
        gemm.scaled_mm(A.float(), B, one, one)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, _fp8((15, 4)), one, one)                          # inner dimensions differ
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, torch.ones(8), one)                            # rowwise scale_a must be (m, 1)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, torch.ones(7, 1), one)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, torch.ones(4, 1))                         # rowwise scale_b must be (1, n)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one.double(), one)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one, out_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one, bias=torch.zeros(4))                 # bf16 out takes a bf16 bias
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one, bias=torch.zeros(5, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one)                                      # CPU tensors
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one, out=torch.empty(8, 4, dtype=torch.bfloat16).t().contiguous().t())
    with pytest.raises(ValueError):                                         # rows of out overlap
        gemm.scaled_mm(A, B, one, one, out=torch.empty(64, dtype=torch.bfloat16).as_strided((8, 4), (2, 1)))
    with pytest.raises(ValueError):
        gemm.scaled_mm(A, B, one, one, out=torch.empty(8, 4, dtype=torch.float16))


@need_torch
def test_scaled_mm_layouts_match_torch_conventions(gemm):
    """torch._scaled_mm's layout, a row-major A and a column-major B (W.t()), is (N, T) and read in place; the others
    resolve as for gemm()."""
    x, W = _fp8((8, 32)), _fp8((16, 32))
    assert gemm.operand_layout(tuple(x.shape), x.stride()) == (OP_N, 32)
    assert gemm.operand_layout(tuple(W.t().shape), W.t().stride()) == (OP_T, 32)
    assert gemm.operand_layout(tuple(x.t().shape), x.t().stride()) == (OP_T, 32)
    with pytest.raises(ValueError):
        gemm.operand_layout((8, 4), (8, 2))


def exact_operands(rng, m, n, k, ta, tb):
    """Integer FP8 operands in [-2, 2] (k <= 500: every partial sum is an integer below 2^11 in magnitude)."""
    assert k <= 500
    a = rng.integers(-2, 3, (m, k)).astype(np.float32)
    b = rng.integers(-2, 3, (k, n)).astype(np.float32)
    return encode(a, ta), encode(b, tb)


@need_torch
def test_oracle_matches_torch_scaled_mm_on_cpu():
    """The numpy oracle equals torch._scaled_mm on the CPU for tensorwise scales on exact products."""
    rng = np.random.default_rng(1)
    m, n, k = 24, 40, 96
    for ta, tb in PAIRS:
        a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        a, b = decode(a8, ta), decode(b8, tb)
        for o in (OUT_F32, OUT_BF16):
            for s_a, s_b in ((1.0, 1.0), (0.5, 4.0), (2.0 ** -3, 0.25)):
                A = torch.from_numpy(a8).view(fp8_dtype(ta))
                Bt = torch.from_numpy(np.ascontiguousarray(b8.T)).view(fp8_dtype(tb))
                try:
                    want = torch._scaled_mm(A, Bt.t(), torch.tensor(s_a), torch.tensor(s_b), out_dtype=out_dtype(o))
                except (RuntimeError, NotImplementedError) as e:
                    pytest.skip(f"torch._scaled_mm has no CPU kernel here: {e}")
                got = oracle(a, b, np.full(m, s_a, np.float32), np.full(n, s_b, np.float32), None, o)
                assert np.array_equal(want.float().numpy(), got), (ta, tb, o, s_a, s_b)


# ==== GPU ==========================================================================================================
@pytest.fixture
def fresh_bn(gemm):
    yield gemm
    gemm.lib.b200_gemm_debug_set_bn(0)


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def run(gemm, a8, b8, ta, tb, sa, sb, bias, o, fast, op_a=OP_N, op_b=OP_T, lda=None, ldb=None, m=None, n=None, k=None,
        ldc=None):
    """b200_gemm_fp8 on device copies: a8 / b8 are the stored bytes (A as given by op_a, B by op_b); sa / sb float32
    (1 element: tensorwise); bias float32 values of the output type, or None.  Returns C as float32 numpy."""
    if m is None:
        m, k = (a8.shape[1], a8.shape[0]) if op_a else a8.shape
        n = b8.shape[0] if op_b else b8.shape[1]
    lda = lda or a8.shape[1]
    ldb = ldb or b8.shape[1]
    ldc = ldc or n
    A, B = dev(a8), dev(b8)
    Sa, Sb = dev(np.asarray(sa, np.float32)), dev(np.asarray(sb, np.float32))
    Bi = torch.from_numpy(bias).to(out_dtype(o)).cuda() if bias is not None else None
    Cm = torch.full((max(m, 1), ldc), float("nan"), dtype=out_dtype(o), device="cuda")
    rc = gemm.lib.b200_gemm_fp8(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, Sa.data_ptr(),
                                int(Sa.numel() > 1), Sb.data_ptr(), int(Sb.numel() > 1),
                                Bi.data_ptr() if Bi is not None else None, Cm.data_ptr(), ldc, o, fast, None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return Cm[:m, :n].float().cpu().numpy()


def pow2_scales(rng, count):
    return (2.0 ** rng.integers(-3, 4, count)).astype(np.float32)


def same_bits(x, y):
    return np.array_equal(x.view(np.uint32), y.view(np.uint32))


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
@pytest.mark.parametrize("o", [OUT_F32, OUT_BF16, OUT_F16], ids=lambda o: OUT_NAME[o])
@pytest.mark.parametrize("mode", ["fast256", "fast192", "fast128", "promoted"])
def test_exact_class_bit_exact(fresh_bn, pair, o, mode):
    """Every pair, output type, width and accumulation mode equals the oracle bit for bit on exact operands, with M /
    N / K tails, tensorwise and rowwise scales, with and without a bias."""
    gemm = fresh_bn
    ta, tb = pair
    fast = mode != "promoted"
    bn = int(mode[4:]) if fast else 128
    gemm.lib.b200_gemm_debug_set_bn(bn)
    rng = np.random.default_rng(hash((pair, o, mode)) & 0xFFFF)
    for m, n, k in ((200, 300, 300), (129, 257, 129), (64, 40, 32)):
        a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        a, b = decode(a8, ta), decode(b8, tb)
        bt8 = np.ascontiguousarray(b8.T)
        for rowwise in (False, True):
            sa = pow2_scales(rng, m if rowwise else 1)
            sb = pow2_scales(rng, n if rowwise else 1)
            for with_bias in (False, True):
                bias = round_out(rng.integers(-64, 65, n).astype(np.float32) / 8, o) if with_bias else None
                got = run(gemm, a8, bt8, ta, tb, sa, sb, bias, o, int(fast))
                want = oracle(a, b, np.broadcast_to(sa, m), np.broadcast_to(sb, n), bias, o)
                assert same_bits(got, want), (m, n, k, rowwise, with_bias)
                assert gemm.last_kernel() == f"tc_{PAIR_NAME[pair]}_{OUT_NAME[o]}{'' if fast else '_acc'}_128x{bn}"


@gpu
@pytest.mark.parametrize("fast", [0, 1])
def test_layouts_and_pitches_match_nt(gemm, fast):
    """NN, TN and TT, unaligned pitches and unaligned bases are bit-identical to the aligned (N, T) call on copies;
    tensorwise scales are bit-identical to rowwise vectors of that constant."""
    rng = np.random.default_rng(7 + fast)
    m, n, k = 190, 250, 333
    ta, tb = E4M3, E5M2
    a = rng.standard_normal((m, k)).astype(np.float32)
    b = rng.standard_normal((k, n)).astype(np.float32)
    a8, b8 = encode(a, ta), encode(b, tb)
    sa, sb = np.float32([0.75]), np.float32([1.5])
    bias = round_out(rng.standard_normal(n).astype(np.float32), OUT_BF16)
    ref = run(gemm, a8, np.ascontiguousarray(b8.T), ta, tb, sa, sb, bias, OUT_BF16, fast)
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            sa8 = np.ascontiguousarray(a8.T) if op_a else a8
            sb8 = np.ascontiguousarray(b8.T) if op_b else b8
            got = run(gemm, sa8, sb8, ta, tb, sa, sb, bias, OUT_BF16, fast, op_a, op_b)
            assert same_bits(got, ref), (op_a, op_b)
    # unaligned pitch (ld % 16 != 0) and base (one byte in) for the (N, T) layout
    for pad, off in ((3, 0), (0, 1), (5, 1)):
        A = np.zeros((m, k + pad + off), np.uint8)
        A[:, off:off + k] = a8
        Bt = np.zeros((n, k + pad + off), np.uint8)
        Bt[:, off:off + k] = b8.T
        Ad, Bd = dev(A), dev(Bt)
        Sa, Sb = dev(sa), dev(sb)
        Bi = torch.from_numpy(bias).to(torch.bfloat16).cuda()
        Cm = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
        rc = gemm.lib.b200_gemm_fp8(OP_N, OP_T, ta, tb, m, n, k, Ad.data_ptr() + off, k + pad + off, Bd.data_ptr() + off,
                                    k + pad + off, Sa.data_ptr(), 0, Sb.data_ptr(), 0, Bi.data_ptr(), Cm.data_ptr(), n,
                                    OUT_BF16, fast, None)
        assert rc == 0
        assert same_bits(Cm.float().cpu().numpy(), ref), (pad, off)
    rows = run(gemm, a8, np.ascontiguousarray(b8.T), ta, tb, np.full(m, sa[0], np.float32), np.full(n, sb[0], np.float32),
               bias, OUT_BF16, fast)
    assert same_bits(rows, ref)


# ---- precision ------------------------------------------------------------------------------------------------------
def crafted_sum(gemm, big_exp, split, fast):
    """acc of one output element: 2^big_exp (an e4m3 power of two up to 2^8 times an e5m2 one up to 2^15) at K index 0,
    then +1 at K index `split` (in the same MMA for split < 32, a later one otherwise).  Ordinary finite inputs.
    Returns the fp32 result minus 2^big_exp."""
    k = 128
    a = np.zeros((1, k), np.float32)
    b = np.zeros((k, 1), np.float32)
    e1 = min(big_exp, 8)
    a[0, 0], b[0, 0] = 2.0 ** e1, 2.0 ** (big_exp - e1)
    a[0, split], b[split, 0] = 1.0, 1.0
    a8, b8 = encode(a, E4M3), encode(b, E5M2)
    c = run(gemm, a8, np.ascontiguousarray(b8.T), E4M3, E5M2, np.float32([1]), np.float32([1]), None, OUT_F32, fast)
    return float(c[0, 0]) - 2.0 ** big_exp


def retained_bits(gemm, split, fast=1):
    """Largest p such that 2^(p-1) + 1 is kept exactly by the tensor core's FP8 accumulation."""
    p = 1
    while p < 24 and crafted_sum(gemm, p, split, fast) == 1.0:
        p += 1
    return p


@gpu
def test_retained_accumulation_precision(gemm):
    """The tensor core keeps RETAINED_BITS significant bits when it adds FP8 products into its accumulator (inside one
    MMA and across MMAs); the promoted mode's chunk of 128 elements is what bounds the error.  The fp32 exact
    representation would keep 24."""
    inside, across = retained_bits(gemm, 1), retained_bits(gemm, 64)
    print(f"retained FP8 accumulation bits: inside one MMA {inside}, across MMAs {across}")
    assert min(inside, across) >= RETAINED_BITS, (inside, across)


def rel_err_bound_promoted(k):
    """|acc - exact| <= bound * sum_k |a_k b_k|.  Inside each 128-element chunk the tensor core's CHUNK / 32 MMAs each
    lose at most two truncations at RETAINED_BITS bits (aligning the MMA's products, then adding them to the chunk's
    accumulator), each at most 2^(1 - RETAINED_BITS) of a magnitude no larger than the chunk's sum of |products|; then
    ceil(k / 128) - 1 rounded fp32 adds of the running sum, each at most 2^-24 of a magnitude no larger than the whole
    sum of |products|."""
    chunks = -(-k // CHUNK)
    return (CHUNK // 32) * 2 * 2.0 ** (1 - RETAINED_BITS) + chunks * 2.0 ** -24


@gpu
@pytest.mark.parametrize("k", [1024, 4096, 16384])
def test_promoted_precision_on_random_operands(gemm, k):
    """Random e4m3 operands: the promoted error stays inside the derived bound, is no larger than fast-accum's on the
    same inputs, and is within 2x of torch._scaled_mm(use_fast_accum=False)'s on the same card."""
    rng = np.random.default_rng(k)
    m, n = 256, 256
    a8 = encode(rng.standard_normal((m, k)) * 4, E4M3)
    b8 = encode(rng.standard_normal((k, n)) * 4, E4M3)
    a, b = decode(a8, E4M3).astype(np.float64), decode(b8, E4M3).astype(np.float64)
    exact = a @ b
    mag = np.abs(a) @ np.abs(b)
    bt8 = np.ascontiguousarray(b8.T)
    one = np.float32([1])
    prom = run(gemm, a8, bt8, E4M3, E4M3, one, one, None, OUT_F32, 0)
    fast = run(gemm, a8, bt8, E4M3, E4M3, one, one, None, OUT_F32, 1)
    err_p = np.abs(prom - exact)
    err_f = np.abs(fast - exact)
    bound = rel_err_bound_promoted(k) * mag
    assert np.all(err_p <= bound), float((err_p / mag).max())
    assert err_p.max() <= err_f.max(), (err_p.max(), err_f.max())
    A = dev(a8).view(torch.float8_e4m3fn)
    Bt = dev(bt8).view(torch.float8_e4m3fn)
    s1 = torch.ones((), device="cuda")
    t = torch._scaled_mm(A, Bt.t(), s1, s1, out_dtype=torch.float32, use_fast_accum=False).cpu().numpy()
    err_t = np.abs(t - exact)
    print(f"k={k}: max |err| / sum|ab|: promoted {(err_p / mag).max():.3e}, fast {(err_f / mag).max():.3e}, "
          f"torch {(err_t / mag).max():.3e}; max |err|: {err_p.max():.4g} / {err_f.max():.4g} / {err_t.max():.4g}")
    assert err_p.max() <= 2 * err_t.max() + 1e-6 * mag.max()


# ---- non-finite values ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
@pytest.mark.parametrize("fast", [0, 1])
def test_non_finite_operands_and_scales(gemm, pair, fast):
    """NaN in either operand type and +-inf in e5m2 give non-finite results exactly where IEEE arithmetic does (0 * inf
    is NaN); so do NaN and inf scales.  Elsewhere the result is the exact oracle."""
    ta, tb = pair
    rng = np.random.default_rng(11 + fast)
    m, n, k = 96, 80, 200
    a8, b8 = exact_operands(rng, m, n, k, ta, tb)
    a, b = decode(a8, ta), decode(b8, tb)
    specials = [np.nan] + ([np.inf, -np.inf] if ta == E5M2 else [])
    for i, v in enumerate(specials):
        a[3 + 7 * i, 5 + i] = v
    specials_b = [np.nan] + ([np.inf, -np.inf] if tb == E5M2 else [])
    for i, v in enumerate(specials_b):
        b[9 + i, 11 + 5 * i] = v
    b[:, 20] = 0.0                                    # inf * 0 = NaN in this column
    b[140, :] = 0.0
    if ta == E5M2:
        a[50, 140] = np.inf                           # row 50 meets the zero row of B: NaN across it
    a8, b8 = encode(a, ta), encode(b, tb)
    a, b = decode(a8, ta), decode(b8, tb)
    sa = pow2_scales(rng, m)
    sb = pow2_scales(rng, n)
    sa[60], sa[61], sb[30] = np.nan, np.inf, -np.inf
    with np.errstate(invalid="ignore"):
        want = oracle(a, b, sa, sb, None, OUT_F32)
    got = run(gemm, a8, np.ascontiguousarray(b8.T), ta, tb, sa, sb, None, OUT_F32, fast)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = ~np.isnan(want)
    assert np.array_equal(got[fin], want[fin])
    assert np.isnan(want).any() and np.isinf(want).any()


@gpu
def test_fp16_output_overflows_to_inf(gemm):
    m, n, k = 64, 64, 64
    a8 = encode(np.full((m, k), 16.0), E4M3)
    b8 = encode(np.full((n, k), 16.0), E4M3)
    got = run(gemm, a8, b8, E4M3, E4M3, np.float32([4]), np.float32([-4]), None, OUT_F16, 0)  # 16384 * 16 = 2^18
    assert np.all(got == -np.inf)


# ---- degenerate shapes ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("o", [OUT_F32, OUT_BF16, OUT_F16], ids=lambda o: OUT_NAME[o])
def test_k_zero_and_empty(gemm, o):
    """k == 0 stores round_out(+0 + bias_j), or +0 (raw zero bits); m == 0 or n == 0 writes nothing."""
    m, n = 70, 50
    for with_bias in (False, True):
        bias = np.linspace(-3, 3, n).astype(np.float32)
        bias[0] = -0.0
        bias = round_out(bias, o)
        Bi = torch.from_numpy(bias).to(out_dtype(o)).cuda() if with_bias else None
        Cm = torch.full((m, n), float("nan"), dtype=out_dtype(o), device="cuda")
        one = torch.ones(1, device="cuda")
        rc = gemm.lib.b200_gemm_fp8(OP_N, OP_T, E4M3, E4M3, m, n, 0, None, 0, None, 0, one.data_ptr(), 0, one.data_ptr(),
                                    0, Bi.data_ptr() if with_bias else None, Cm.data_ptr(), n, o, 0, None)
        assert rc == 0
        got = Cm.float().cpu().numpy()
        want = np.broadcast_to((np.float32(0) + bias) if with_bias else np.float32(0), (m, n))
        assert same_bits(np.ascontiguousarray(got), np.ascontiguousarray(want).astype(np.float32))
    for mm, nn in ((0, n), (m, 0)):
        Cm = torch.full((m, n), 7.0, dtype=out_dtype(o), device="cuda")
        rc = gemm.lib.b200_gemm_fp8(OP_N, OP_T, E4M3, E4M3, mm, nn, 16, None, 16, None, 16, None, 0, None, 0, None,
                                    Cm.data_ptr(), n, o, 0, None)
        assert rc == 0
        assert bool((Cm == 7).all())


# ---- scaled_mm against torch._scaled_mm ----------------------------------------------------------------------------
def torch_combos():
    """(ta, tb, rowwise, out) combinations to try against torch._scaled_mm (those torch refuses are skipped)."""
    for ta, tb in PAIRS:
        for o in (OUT_BF16, OUT_F16, OUT_F32):
            yield ta, tb, False, o
        yield ta, tb, True, OUT_BF16


@gpu
@pytest.mark.parametrize("combo", list(torch_combos()), ids=lambda c: f"{PAIR_NAME[c[:2]]}-{'row' if c[2] else 'tensor'}-"
                                                                     f"{OUT_NAME[c[3]]}")
@pytest.mark.parametrize("fast", [False, True])
def test_scaled_mm_matches_torch(gemm, combo, fast):
    """scaled_mm equals torch._scaled_mm bit for bit on exact operands, for every combination torch accepts."""
    ta, tb, rowwise, o = combo
    rng = np.random.default_rng(3)
    m, n, k = 192, 320, 384
    a8, b8 = exact_operands(rng, m, n, k, ta, tb)
    A = dev(a8).view(fp8_dtype(ta))
    W = dev(np.ascontiguousarray(b8.T)).view(fp8_dtype(tb))         # (n, k): B = W.t()
    sa = dev(pow2_scales(rng, m).reshape(m, 1) if rowwise else pow2_scales(rng, 1).reshape(()))
    sb = dev(pow2_scales(rng, n).reshape(1, n) if rowwise else pow2_scales(rng, 1).reshape(()))
    bias = torch.from_numpy(rng.integers(-8, 9, n).astype(np.float32) / 4).to(out_dtype(o)).cuda()
    for bi in (None, bias):
        try:
            want = torch._scaled_mm(A, W.t(), sa, sb, bias=bi, out_dtype=out_dtype(o), use_fast_accum=fast)
        except (RuntimeError, NotImplementedError) as e:
            pytest.skip(f"torch._scaled_mm refuses this combination: {str(e).splitlines()[0]}")
        got = gemm.scaled_mm(A, W.t(), sa, sb, bias=bi, out_dtype=out_dtype(o), use_fast_accum=fast)
        assert got.dtype == want.dtype and got.shape == want.shape
        assert same_bits(got.float().cpu().numpy(), want.float().cpu().numpy()), bi is None


@gpu
@pytest.mark.parametrize("fast", [False, True])
def test_scaled_mm_mlp_shape(gemm, fast):
    """An MLP-sized NT call (x @ W.t(), rowwise scales, bf16 out) against torch._scaled_mm and the fp64 product: inside
    the promoted bound plus one bf16 rounding."""
    rng = np.random.default_rng(5)
    m, n, k = 2048, 4096, 4096
    x = torch.from_numpy(rng.standard_normal((m, k)).astype(np.float32)).cuda()
    Wf = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).cuda()
    sx = (x.abs().amax(dim=1, keepdim=True) / 448).float()
    sw = (Wf.abs().amax(dim=1, keepdim=True) / 448).float()
    xq = (x / sx).to(torch.float8_e4m3fn)
    wq = (Wf / sw).to(torch.float8_e4m3fn)
    got = gemm.scaled_mm(xq, wq.t(), sx, sw.t(), out_dtype=torch.bfloat16, use_fast_accum=fast).double()
    want = torch._scaled_mm(xq, wq.t(), sx, sw.t(), out_dtype=torch.bfloat16, use_fast_accum=fast).double()
    exact = (xq.double() * sx.double()) @ (wq.double() * sw.double()).t()
    mag = (xq.double().abs() * sx.double()) @ (wq.double().abs() * sw.double()).t()
    lim = (rel_err_bound_promoted(k) if not fast else 2.0 ** -8) * mag + 2.0 ** -8 * exact.abs()
    if not fast:
        assert bool(((got - exact).abs() <= lim).all())
    err_g, err_w = (got - exact).abs().max().item(), (want - exact).abs().max().item()
    print(f"MLP {m}x{n}x{k} fast={fast}: max |err| ours {err_g:.4g}, torch {err_w:.4g}")
    assert err_g <= 2 * err_w + 1e-6


@gpu
def test_scaled_mm_cuda_graph_with_rewritten_scales(gemm):
    """One capture, replayed with the scale tensors rewritten in place between replays: the host never reads them."""
    rng = np.random.default_rng(9)
    m, n, k = 256, 384, 256
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    a, b = decode(a8, E4M3), decode(b8, E4M3)
    A = dev(a8).view(torch.float8_e4m3fn)
    W = dev(np.ascontiguousarray(b8.T)).view(torch.float8_e4m3fn)
    sa = torch.ones((m, 1), device="cuda")
    sb = torch.ones((1, n), device="cuda")
    out = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gemm.scaled_mm(A, W.t(), sa, sb, out=out, stream=s)         # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gemm.scaled_mm(A, W.t(), sa, sb, out=out)
    for r in range(3):
        va, vb = pow2_scales(rng, m), pow2_scales(rng, n)
        sa.copy_(torch.from_numpy(va).reshape(m, 1))
        sb.copy_(torch.from_numpy(vb).reshape(1, n))
        g.replay()
        torch.cuda.synchronize()
        assert same_bits(out.float().cpu().numpy(), oracle(a, b, va, vb, None, OUT_BF16)), r
