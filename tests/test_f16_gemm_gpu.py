"""IEEE fp16 operands (b200_gemm_f16, b200_gemm_f16_ex) and the general alpha / beta epilogue of the 16-bit GEMMs
(b200_gemm_bf16_ex, b200_gemm_f16_ex).

The fp16 GEMM is the bf16 kernel with the other wgmma type: the same 64-element k-block (one 128-byte row), the same
three tile widths, the same routes and the same split-tail rule (fp32 C may take it, 16-bit C never does), so its
shapes come from the schedule model of test_tile_schedules_gpu.py for bf16 and its layouts are checked the way
test_transposed_ops_gpu.py checks bf16.  Known answers use small dyadic operands, so that every product and every
partial sum is exact in fp32 whatever the accumulation order: fp32 C must equal the exact product bit for bit and
16-bit C its round-to-nearest-even rounding.  Output buffers start as NaN and whole buffers are compared.

The argument checks need no GPU."""
import ctypes as C

import pytest

import test_tile_schedules_gpu as ts
import test_transposed_ops_gpu as tr
from test_transposed_ops_gpu import hooks, sms  # noqa: F401  (fixtures: scheduling hooks reset, SM count)

try:
    import torch
except ImportError:          # the CPU tests need no torch
    torch = None

gpu = pytest.mark.gpu
OP_N, OP_T = tr.OP_N, tr.OP_T
OUT_F32, OUT_BF16, OUT_F16 = 0, 1, 2
LAYS = ("nn", "nt", "tn", "tt")
OPS = {"nn": (OP_N, OP_N), **tr.LAYOUTS}

# kind: (operand dtype, C dtype, out_type, kernel name prefix, schedule-model kind)
KINDS16 = {
    "f16": ("float16", "float32", OUT_F32, "tc_f16", "bf16"),
    "f16_of16": ("float16", "float16", OUT_F16, "tc_f16_of16", "bf16_obf16"),
    "bf16": ("bfloat16", "float32", OUT_F32, "tc_bf16", "bf16"),
    "bf16_obf16": ("bfloat16", "bfloat16", OUT_BF16, "tc_bf16_obf16", "bf16_obf16"),
}
GENERIC = {"float16": "generic_f16_64x64", "bfloat16": "generic_bf16_64x64"}
# the fp16 kernel's schedule: bf16's, per C type (TcConfig: BK = 128 bytes / 2; OutBytes<float> = 4, <f16_out> = 2)
F16_SCHEDULE = {"f16": ts.Kind(64, 4, (128, 192, 256), "tc_f16"), "f16_of16": ts.Kind(64, 2, (128, 192, 256), "tc_f16_of16")}


def test_f16_shares_the_bf16_schedule():
    for kind, kd in F16_SCHEDULE.items():
        ref = ts.KINDS[KINDS16[kind][4]]
        assert (kd.bk, kd.out_bytes, kd.widths) == (ref.bk, ref.out_bytes, ref.widths), kind


# ==== argument checks (no GPU: every case returns before the device is touched) ===============================
def test_f16_argument_validation(gemm):
    lib = gemm.lib
    buf = (C.c_float * 256)()
    m, n, k = 4, 6, 8
    f16 = lambda ot, mm=m, a=buf, lda=k, ldb=n, c=buf: lib.b200_gemm_f16(mm, n, k, a, lda, buf, ldb, c, n, ot, None)
    f16ex = lambda opa, opb, ot, lda, ldb, mm=m, al=0.5, a=buf, c=buf: lib.b200_gemm_f16_ex(
        opa, opb, mm, n, k, al, a, lda, buf, ldb, 0.25, c, n, ot, None)
    bf16ex = lambda opa, opb, ot, lda, ldb, mm=m, al=0.5, a=buf, c=buf: lib.b200_gemm_bf16_ex(
        opa, opb, mm, n, k, al, a, lda, buf, ldb, 0.25, c, n, ot, None)
    # out_type pairings: refused ones before anything else; accepted ones reach the empty-problem no-op (m = 0)
    for ot in (OUT_F32, OUT_BF16, OUT_F16, 3, -1, 7):
        want_f16 = 0 if ot in (OUT_F32, OUT_F16) else -1
        want_bf16 = 0 if ot in (OUT_F32, OUT_BF16) else -1
        assert f16(ot, mm=0) == want_f16, ot
        for al in (1.0, 0.5, 0.0):                      # (1, beta) with beta != 0 and the general pairs alike
            assert f16ex(OP_N, OP_T, ot, k, k, mm=0, al=al) == want_f16, (ot, al)
            assert bf16ex(OP_T, OP_N, ot, m, n, mm=0, al=al) == want_bf16, (ot, al)
        assert lib.b200_gemm_f16_ex(OP_N, OP_N, 0, n, k, 1.0, buf, k, buf, n, 0.0, buf, n, ot, None) == want_f16
        assert lib.b200_gemm_bf16_ex(OP_N, OP_N, 0, n, k, 1.0, buf, k, buf, n, 0.0, buf, n, ot, None) == want_bf16
    for fn, ot in ((f16ex, OUT_F16), (bf16ex, OUT_BF16)):
        for al in (1.0, 0.5):
            for bad in ((2, 0), (0, 2), (-1, 0), (0, -1)):
                assert fn(bad[0], bad[1], ot, 16, 16, al=al) == -1, bad
                assert fn(bad[0], bad[1], ot, 16, 16, mm=0, al=al) == -1, bad          # refused even when empty
            # op-dependent minimum ld: A needs k (N) or m (T), B needs n (N) or k (T)
            assert fn(OP_N, OP_N, ot, k - 1, n, al=al) == -1 and fn(OP_T, OP_N, ot, m - 1, n, al=al) == -1
            assert fn(OP_N, OP_N, ot, k, n - 1, al=al) == -1 and fn(OP_N, OP_T, ot, k, k - 1, al=al) == -1
            assert fn(OP_T, OP_T, ot, m - 1, k, al=al) == -1 and fn(OP_T, OP_T, ot, m, k - 1, al=al) == -1
            assert fn(OP_N, OP_N, ot, k, n, a=None, al=al) == -1                       # null A
            assert fn(OP_N, OP_N, ot, k, n, c=None, al=al) == -1                       # null C
    assert f16(OUT_F16, lda=k - 1) == -1 and f16(OUT_F16, ldb=n - 1) == -1
    assert f16(OUT_F32, a=None) == -1 and f16(OUT_F32, c=None) == -1
    assert lib.b200_gemm_f16(-1, n, k, buf, k, buf, n, buf, n, OUT_F32, None) == -1
    # empty problems are no-ops, null pointers included
    assert lib.b200_gemm_f16(0, n, k, None, 1, None, 1, None, 1, OUT_F16, None) == 0
    assert lib.b200_gemm_f16_ex(OP_T, OP_T, m, 0, k, 0.5, None, 1, None, 1, 2.0, None, 1, OUT_F16, None) == 0
    assert lib.b200_gemm_bf16_ex(OP_N, OP_T, 0, n, k, 0.0, None, 1, None, 1, 0.0, None, 1, OUT_BF16, None) == 0


# ==== GPU helpers ===============================================================================================
def dt(name):
    return getattr(torch, name)


def out_buf16(kind, m, n, c0=None):
    """NaN-filled C of the kind's type with padding columns; c0 (if given) in the first n columns."""
    buf = torch.full((m, n + 1 + n % 2), float("nan"), dtype=dt(KINDS16[kind][1]), device="cuda")
    if c0 is not None:
        buf[:, :n] = c0
    return buf


def call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, k, alpha=1.0, beta=0.0, entry="ex"):
    """One call into buf[:, :n]; returns (launches issued, kernel name).  entry "ex": b200_gemm_f16_ex / _bf16_ex;
    "plain": the call that exists without alpha / beta (b200_gemm_f16, NN only, or b200_gemm_bf16_op)."""
    lib = gemm.lib
    ind, _, ot, _, _ = KINDS16[kind]
    m, ldc = buf.shape[0], buf.stride(0)
    a, b = (Av.data_ptr() if Av is not None else None), (Bv.data_ptr() if Bv is not None else None)
    before = lib.b200_gemm_launch_count()
    if entry == "plain" and ind == "float16":
        assert op_a == OP_N and op_b == OP_N
        rc = lib.b200_gemm_f16(m, n, k, a, lda, b, ldb, buf.data_ptr(), ldc, ot, None)
    elif entry == "plain":
        rc = lib.b200_gemm_bf16_op(op_a, op_b, m, n, k, a, lda, b, ldb, buf.data_ptr(), ldc, ot, None)
    else:
        fn = lib.b200_gemm_f16_ex if ind == "float16" else lib.b200_gemm_bf16_ex
        rc = fn(op_a, op_b, m, n, k, alpha, a, lda, b, ldb, beta, buf.data_ptr(), ldc, ot, None)
    assert rc == 0, (kind, rc)
    return lib.b200_gemm_launch_count() - before, gemm.last_kernel()


def route16(kind, lay, bn, aligned):
    ind, _, _, prefix, _ = KINDS16[kind]
    if not aligned:
        return 1, GENERIC[ind]
    return 1, f"{prefix}{'' if lay == 'nn' else '_' + lay}_128x{bn}"


def logical16(kind, m, n, k, seed, dyadic=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dyadic:               # j / 8, |j| <= 8: every product a multiple of 2^-6, every partial sum exact in fp32
        A = torch.randint(-8, 9, (m, k), device="cuda", generator=g).float() / 8
        B = torch.randint(-8, 9, (k, n), device="cuda", generator=g).float() / 8
    else:
        A = torch.rand((m, k), device="cuda", generator=g) * 2 - 1
        B = torch.rand((k, n), device="cuda", generator=g) * 2 - 1
    d = dt(KINDS16[kind][0])
    return A.to(d), B.to(d)


def run_layouts(gemm, kind, A, B, aligned, bn=None, alpha=1.0, beta=0.0, c0=None, lays=LAYS):
    """Each layout on operands stored as op requires; asserts the route, returns {layout: buf}."""
    m, k = A.shape
    n = B.shape[1]
    res = {}
    for lay in lays:
        op_a, op_b = OPS[lay]
        Av, lda = tr.operand(A, op_a, aligned)
        Bv, ldb = tr.operand(B, op_b, aligned)
        buf = out_buf16(kind, m, n, c0)
        got = call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, k, alpha, beta)
        if bn is not None:
            assert got == route16(kind, lay, bn, aligned), (kind, lay, got)
        assert bool(torch.isnan(buf[:, n:]).all()), (kind, lay)
        res[lay] = buf
    return res


def check_ref16(kind, A, B, got, alpha=1.0, beta=0.0, c0=None):
    """Within ts.TOL["bf16"] of the scale of the float64 answer, plus one rounding of a 16-bit C."""
    t = alpha * (A.double() @ B.double())
    scale = abs(alpha) * float((A.double().abs() @ B.double().abs()).max())
    if c0 is not None and beta != 0.0:
        t = t + beta * c0.double()
        scale += abs(beta) * float(c0.double().abs().max())
    cd = KINDS16[kind][1]
    rel = {"float32": 0.0, "float16": 2.0 ** -11, "bfloat16": 2.0 ** -8}[cd]
    err = (got.double() - t).abs() - t.abs() * rel
    assert float(err.max()) <= ts.TOL["bf16"] * scale, (kind, float(err.max()) / scale)


def shapes16(sms, splits=(2,)):
    """Forced widths with M / N / K tails and ld > dim, then K-split tails of the fp32-C schedule.  (m, n, k, bn)"""
    out = [c for c in ts.width_cases("bf16") if (c[0], c[1] - c[3]) in ((1, -8), (129, 8), (389, c[3] + 8))]
    return out + [ts.split_case("bf16", s, sms, False) for s in splits]


def splits_of(kind, m, n, k, bn, sms):
    return ts.tc_split(m, n, k, KINDS16[kind][4], bn, sms)


# ==== 1. known answers ==========================================================================================
@gpu
@pytest.mark.parametrize("kind", ["f16", "f16_of16"])
def test_known_answers_bit_exact(gemm, hooks, sms, kind):
    """Dyadic fp16 operands: fp32 C is the exact product and fp16 C its RNE rounding, bit for bit, in every layout,
    every forced width, with M / N / K tails and (fp32 C) K-split tails of 2, 3 and 4 parts."""
    seen_split = set()
    for i, (m, n, k, bn) in enumerate(shapes16(sms, (2, 3, 4))):
        hooks.b200_gemm_debug_set_bn(bn)
        seen_split.add(splits_of(kind, m, n, k, bn, sms))
        A, B = logical16(kind, m, n, k, 100 + i, dyadic=True)
        exact = (A.double() @ B.double()).float()          # exact in fp32 (|sum| < 2^18 in steps of 2^-6)
        want = exact.to(dt(KINDS16[kind][1]))
        for lay, buf in run_layouts(gemm, kind, A, B, True, bn).items():
            assert tr.same_bits(buf[:, :n], want), (kind, lay, (m, n, k, bn))
    assert seen_split == ({1, 2, 3, 4} if kind == "f16" else {1})


# ==== 2. layouts against NN, routes, the float64 reference =====================================================
@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
@pytest.mark.parametrize("kind", ["f16", "f16_of16"])
def test_layouts_bit_identical_to_nn(gemm, hooks, sms, kind, aligned):
    for i, (m, n, k, bn) in enumerate(shapes16(sms)):
        hooks.b200_gemm_debug_set_bn(bn)
        A, B = logical16(kind, m, n, k, 200 + i)
        res = run_layouts(gemm, kind, A, B, aligned, bn)
        for lay in LAYS[1:]:
            assert tr.same_bits(res[lay], res["nn"]), (kind, lay, (m, n, k, bn), aligned)
        check_ref16(kind, A, B, res["nn"][:, :n])


# ==== 3. output rounding: 16-bit C is the RNE rounding of the fp32-C result ====================================
@gpu
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-0.75, 0.5)] + ts.EXTREMES,
                         ids=["plain", "general", "tiny_alpha", "tiny_beta", "pow2"])
@pytest.mark.parametrize("ind", ["float16", "bfloat16"])
def test_16bit_c_is_rounded_fp32_c(gemm, hooks, sms, ind, alpha, beta):
    """With the split tail off both C types accumulate in the same order, and beta * C reads the same value (fp32 C
    seeded with float(C16)), so the 16-bit result must be the RNE rounding of the fp32 one, overflow to inf included
    (fp16 C under beta = 1e20).  Tensor-core and generic routes, every layout."""
    hooks.b200_gemm_debug_set_split_tail(0)
    k32, k16 = ("f16", "f16_of16") if ind == "float16" else ("bf16", "bf16_obf16")
    m, n, k, bn = ts.split_case("bf16", 2, sms, False)
    hooks.b200_gemm_debug_set_bn(bn)
    A, B = logical16(k32, m, n, k, 300)
    g = torch.Generator(device="cuda").manual_seed(301)
    c16 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(dt(ind))
    for aligned in (True, False):
        r32 = run_layouts(gemm, k32, A, B, aligned, bn, alpha, beta, c16.float())
        r16 = run_layouts(gemm, k16, A, B, aligned, bn, alpha, beta, c16)
        for lay in LAYS:
            assert tr.same_bits(r16[lay][:, :n], r32[lay][:, :n].to(dt(ind))), (ind, lay, aligned, alpha, beta)


# ==== 4. alpha / beta ===========================================================================================
@gpu
@pytest.mark.parametrize("alpha,beta", [(-0.75, 0.5), (1.0, 1.0)] + ts.EXTREMES,
                         ids=["general", "one_one", "tiny_alpha", "tiny_beta", "pow2"])
@pytest.mark.parametrize("kind", list(KINDS16))
def test_alpha_beta(gemm, hooks, sms, kind, alpha, beta):
    """C = alpha op(A) op(B) + beta C in every layout, on the tensor cores (fp32 C with a K-split tail: beta * C is
    folded by part 0) and on the generic kernel: bit-identical to NN, within tolerance of the float64 answer."""
    m, n, k, bn = ts.split_case("bf16", 2, sms, False)
    assert splits_of(kind, m, n, k, bn, sms) == (2 if KINDS16[kind][1] == "float32" else 1)
    hooks.b200_gemm_debug_set_bn(bn)
    A, B = logical16(kind, m, n, k, 400)
    g = torch.Generator(device="cuda").manual_seed(401)
    c0 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(dt(KINDS16[kind][1]))
    for aligned in (True, False):
        res = run_layouts(gemm, kind, A, B, aligned, bn, alpha, beta, c0)
        for lay in LAYS[1:]:
            assert tr.same_bits(res[lay], res["nn"]), (kind, lay, aligned)
        got = res["nn"][:, :n]
        if kind == "f16_of16" and max(abs(alpha), abs(beta)) > 65504:
            assert bool(torch.isinf(got).any())           # beyond the fp16 range: +-inf (test 3 pins the bits)
            continue
        assert bool(torch.isfinite(got).all())
        check_ref16(kind, A, B, got, alpha, beta, c0)


@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_alpha_beta_zero_rules(gemm, hooks, sms, kind):
    """alpha == 0 never reads A or B (NaN operands; one element-wise pass C = round(beta * float(C)), zeros for
    beta == 0); beta == 0 never reads C (NaN C leaves no trace); k == 0 is C = round(beta * float(C))."""
    m, n, k = 200, 136, 264
    cd = dt(KINDS16[kind][1])
    A, B = logical16(kind, m, n, k, 500)
    g = torch.Generator(device="cuda").manual_seed(501)
    c0 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(cd)
    An, Bn = torch.full_like(A, float("nan")), torch.full_like(B, float("nan"))
    for aligned in (True, False):
        for lay in LAYS:
            op_a, op_b = OPS[lay]
            Av, lda = tr.operand(An, op_a, aligned)
            Bv, ldb = tr.operand(Bn, op_b, aligned)
            for beta in (0.5, 0.0):                      # alpha = 0: A and B are NaN and must not be read
                buf = out_buf16(kind, m, n, c0)
                launches, _ = call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, k, 0.0, beta)
                assert launches == 1
                want = (beta * c0.float()).to(cd) if beta != 0 else torch.zeros_like(c0)     # beta == 0: +0, C unread
                assert tr.same_bits(buf[:, :n], want), (kind, lay, beta)
                assert bool(torch.isnan(buf[:, n:]).all())
            buf = out_buf16(kind, m, n, c0)                # k = 0
            call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, 0, 1.0, -2.0)
            assert tr.same_bits(buf[:, :n], (-2.0 * c0.float()).to(cd))
            Av, lda = tr.operand(A, op_a, aligned)       # beta = 0: C is NaN and must not be read
            Bv, ldb = tr.operand(B, op_b, aligned)
            b_nan, b_zero = out_buf16(kind, m, n), out_buf16(kind, m, n, torch.zeros_like(c0))
            call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b_nan, n, k, -0.75, 0.0)
            call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b_zero, n, k, -0.75, 0.0)
            assert bool(torch.isfinite(b_nan[:, :n]).all()) and tr.same_bits(b_nan, b_zero), (kind, lay, aligned)


@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_ex_one_zero_is_the_plain_call(gemm, hooks, sms, kind):
    """(alpha, beta) = (1, 0) through _ex: the bits, kernel name and launch count of b200_gemm_f16 / _bf16_op."""
    m, n, k, bn = ts.split_case("bf16", 2, sms, False)
    A, B = logical16(kind, m, n, k, 600)
    lays = ("nn",) if KINDS16[kind][0] == "float16" else LAYS
    for aligned in (True, False):
        for lay in lays:
            op_a, op_b = OPS[lay]
            Av, lda = tr.operand(A, op_a, aligned)
            Bv, ldb = tr.operand(B, op_b, aligned)
            b1, b2 = out_buf16(kind, m, n), out_buf16(kind, m, n)
            r1 = call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b1, n, k, entry="plain")
            r2 = call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b2, n, k, 1.0, 0.0)
            assert r1 == r2 and tr.same_bits(b1, b2), (kind, lay, aligned, r1, r2)


# ==== 5. range ====================================================================================================
@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
def test_fp16_subnormal_operands_are_kept(gemm, aligned):
    """A = j * 2^-24 (fp16 subnormals down to the smallest, 2^-24), B small integers: the products are exact in
    fp32 and nothing may be flushed to zero."""
    m, n, k = 136, 200, 264
    g = torch.Generator(device="cuda").manual_seed(700)
    A = (torch.randint(-1023, 1024, (m, k), device="cuda", generator=g).double() * 2.0 ** -24)
    A[:, 0] = 2.0 ** -24
    B = torch.randint(-4, 5, (k, n), device="cuda", generator=g).double()
    B[0, :] = 1.0
    exact = (A @ B).float()
    for lay in LAYS:
        res = run_layouts(gemm, "f16", A.half(), B.half(), aligned, lays=(lay,))
        assert tr.same_bits(res[lay][:, :n], exact), lay
        assert bool((res[lay][:, :n] != 0).any())


@gpu
@pytest.mark.parametrize("kind", ["f16", "f16_of16"])
def test_nonfinite_operands_stay_in_their_row_and_column(gemm, kind):
    m, n, k = 200, 136, 264
    A, B = logical16(kind, m, n, k, 710)
    A[3, 10], A[77, 5], B[9, 100] = float("inf"), float("nan"), float("-inf")
    want = torch.zeros((m, n), dtype=torch.bool, device="cuda")
    want[3, :], want[77, :], want[:, 100] = True, True, True
    for aligned in (True, False):
        for lay, buf in run_layouts(gemm, kind, A, B, aligned).items():
            assert torch.equal(~torch.isfinite(buf[:, :n]), want), (kind, lay, aligned)


@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
def test_fp16_c_overflows_to_inf(gemm, aligned):
    """fp16 C rounds to nearest even at the top of the range: a true 65519 stores 65504 (the largest fp16), 65520
    (the midpoint to 65536) rounds to even and overflows to inf, as torch's .half() does; fp32 C is exact."""
    x = [1007.0, 1008.0, 992.0, -1008.0, 1200.0, 0.0]       # C(i, 0) = 1024 * 63 + x_i
    want32 = [65519.0, 65520.0, 65504.0, 64512.0 - 1008.0, 65712.0, 64512.0]
    A = torch.tensor([[1024.0, v] for v in x], device="cuda")
    A[3, 0] = -1024.0
    want32[3] = -65520.0
    B = torch.tensor([[63.0] * 8, [1.0] * 8], device="cuda")
    res32 = run_layouts(gemm, "f16", A.half(), B.half(), aligned)
    res16 = run_layouts(gemm, "f16_of16", A.half(), B.half(), aligned)
    inf = float("inf")
    want16 = torch.tensor([65504.0, inf, 65504.0, -inf, inf, 64512.0], device="cuda").half()
    for lay in LAYS:
        assert torch.equal(res32[lay][:, :8], torch.tensor(want32, device="cuda")[:, None].expand(6, 8)), lay
        assert tr.same_bits(res16[lay][:, :8], want16[:, None].expand(6, 8)), lay
        assert tr.same_bits(res16[lay][:, :8], res32[lay][:, :8].half())


# ==== 6. routes ==================================================================================================
@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
@pytest.mark.parametrize("kind", ["f16", "f16_of16"])
def test_routes(gemm, sms, kind, aligned):
    """The fp16 row of the header's launch table: one launch in every layout, the tile width of the heuristic."""
    for m, n, k in ((200, 136, 264), (1000, 3000, 520), (4096, 1024, 128)):
        bn = ts.pick_bn(m, n, sms, "bf16")
        A, B = logical16(kind, m, n, k, 800)
        run_layouts(gemm, kind, A, B, aligned, bn)


# ==== 7. the tensor-level interface ===============================================================================
@gpu
def test_python_gemm_fp16(gemm):
    g = torch.Generator(device="cuda").manual_seed(900)
    x = (torch.rand((300, 520), device="cuda", generator=g) * 2 - 1).half()
    W = (torch.rand((264, 520), device="cuda", generator=g) * 2 - 1).half()       # n x k, as a linear layer holds it
    for out_dtype in (torch.float32, torch.float16):
        want = gemm.gemm(x, W.t().contiguous(), out_dtype=out_dtype)
        assert want.dtype == out_dtype
        out = torch.empty((300, 264), device="cuda", dtype=out_dtype)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        gemm.gemm(x, W.t(), out=out)
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() == before                  # no copy of W was made
        assert gemm.last_kernel() == ("tc_f16_nt_128x128" if out_dtype == torch.float32 else "tc_f16_of16_nt_128x128")
        assert tr.same_bits(out, want)
    assert gemm.gemm(x, W.t()).dtype == torch.float32                            # default C type
    # alpha / beta for fp16 and bf16 against the C entry points
    for ind, fn, ot16 in ((torch.float16, gemm.lib.b200_gemm_f16_ex, OUT_F16), (torch.bfloat16, gemm.lib.b200_gemm_bf16_ex, OUT_BF16)):
        xa, Wa = x.to(ind), W.to(ind)
        for cd, ot in ((torch.float32, OUT_F32), (ind, ot16)):
            c0 = (torch.rand((300, 264), device="cuda", generator=g) * 2 - 1).to(cd)
            o1, o2 = c0.clone(), c0.clone()
            gemm.gemm(xa, Wa.t(), out=o1, alpha=0.5, beta=-2.0)
            assert fn(OP_N, OP_T, 300, 264, 520, 0.5, xa.data_ptr(), 520, Wa.data_ptr(), 520, -2.0, o2.data_ptr(), 264, ot,
                      torch.cuda.current_stream().cuda_stream) == 0
            assert tr.same_bits(o1, o2), (ind, cd)
    # bf16 at (1, 0) keeps its path
    before = gemm.launch_count()
    gemm.gemm(x.bfloat16(), W.bfloat16().t())
    assert gemm.launch_count() - before == 1 and gemm.last_kernel() == "tc_bf16_nt_128x128"
    x8 = torch.randint(-127, 128, (300, 520), device="cuda", generator=g, dtype=torch.int8)
    W8 = torch.randint(-127, 128, (264, 520), device="cuda", generator=g, dtype=torch.int8)
    with pytest.raises(ValueError):
        gemm.gemm(x8, W8.t(), alpha=2.0)                                        # int8 keeps alpha = 1, beta = 0
    with pytest.raises(TypeError):
        gemm.gemm(x, W.bfloat16().t())                                          # mixed fp16 / bf16 operands
    with pytest.raises(AssertionError):
        gemm.gemm(x, W.t(), out_dtype=torch.bfloat16)                           # fp16 operands never write bf16
