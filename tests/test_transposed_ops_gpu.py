"""Transposed operands (B200_OP_T) in the fp32, bf16 and int8 GEMMs: b200_gemm_f32_op, _bf16_op, _s8s32_op.

Every result with a transposed operand must equal, bit for bit, the NN call on row-major copies of op(A) and op(B)
with leading dimensions of the same alignment class: the tensor cores see the same values in the same K order, the
plane split is elementwise and the F16X2 maxima are taken over the same sets whichever pre-pass kernel takes them.
The same cases must lie within the tolerances of test_tile_schedules_gpu.py of a float64 product (int8 exact), the
split modes must keep the range edges of test_fp32_range_gpu.py and the known answers of their exact models, and
the launch count and kernel name of every call show the route it took (B^T read in place, pre-pass roles swapped).
Shapes come from the schedule model of test_tile_schedules_gpu.py.  Output buffers start as NaN (or a sentinel) and
whole buffers are compared.

The argument checks, the workspace sizes and the Python layout resolver need no GPU."""
import ctypes as C

import numpy as np
import pytest

import _fp32_model as fm
import _libs
import test_fp32_range_gpu as fr
import test_tile_schedules_gpu as ts

try:
    import torch
except ImportError:          # the CPU tests need no torch
    torch = None

gpu = pytest.mark.gpu
OP_N, OP_T = 0, 1
LAYOUTS = {"nt": (OP_N, OP_T), "tn": (OP_T, OP_N), "tt": (OP_T, OP_T)}
F32_MODES = {"strict": 0, "tf32": 1, "bf16x3": 2, "bf16x2": 3, "auto": 4, "f16x2": 5}


# ==== argument checks and workspace sizes (no GPU: check_args runs before the device check) =================
def test_op_argument_validation(gemm):
    lib = gemm.lib
    buf = (C.c_float * 256)()
    m, n, k = 4, 6, 8
    f32 = lambda opa, opb, lda, ldb, ldc=n, mm=m: lib.b200_gemm_f32_op(opa, opb, mm, n, k, 1.0, buf, lda, buf, ldb, 0.0,
                                                                      buf, ldc, 0, None)
    bf16 = lambda opa, opb, lda, ldb: lib.b200_gemm_bf16_op(opa, opb, m, n, k, buf, lda, buf, ldb, buf, n, 0, None)
    s8 = lambda opa, opb, lda, ldb: lib.b200_gemm_s8s32_op(opa, opb, m, n, k, buf, lda, buf, ldb, buf, n, None)
    for fn in (f32, bf16, s8):
        for bad in ((2, 0), (0, 2), (-1, 0), (0, -1)):
            assert fn(bad[0], bad[1], 16, 16) == -1, (fn, bad)
        # op-dependent minimum ld: A needs k (N) or m (T), B needs n (N) or k (T)
        assert fn(OP_N, OP_N, k - 1, n) == -1 and fn(OP_T, OP_N, m - 1, n) == -1
        assert fn(OP_N, OP_N, k, n - 1) == -1 and fn(OP_N, OP_T, k, k - 1) == -1
        assert fn(OP_T, OP_T, m - 1, k) == -1 and fn(OP_T, OP_T, m, k - 1) == -1
    assert f32(OP_T, OP_T, m, k, ldc=n - 1) == -1                                   # ldc < n
    assert f32(2, OP_N, 16, 16, mm=0) == -1                                         # a bad op is refused even when empty
    assert lib.b200_gemm_bf16_op(OP_N, OP_T, m, n, k, buf, k, buf, k, buf, n, 7, None) == -1    # bad out_type
    assert lib.b200_gemm_f32_op(OP_T, OP_T, 0, n, k, 1.0, None, 1, None, 1, 0.0, None, 1, 0, None) == 0   # empty: no-op
    assert lib.b200_gemm_s8s32_op(OP_T, OP_N, m, 0, k, None, 1, None, 1, None, 1, None) == 0
    assert lib.b200_gemm_bf16_op(OP_N, OP_T, m, n, k, None, k, buf, k, buf, n, 0, None) == -1      # null A
    assert lib.b200_gemm_f32_op(OP_T, OP_N, -1, n, k, 1.0, buf, m, buf, n, 0.0, buf, n, 0, None) == -1


@pytest.mark.parametrize("mode", sorted(F32_MODES.values()))
def test_workspace_bytes_op(gemm, mode):
    lib = gemm.lib
    for m, n, k in ((1, 1, 1), (200, 136, 264), (4096, 4096, 4096), (1000, 3000, 77), (129, 520, 1025)):
        assert lib.b200_gemm_workspace_bytes_op(OP_N, OP_N, m, n, k, mode) == lib.b200_gemm_workspace_bytes(m, n, k, mode)
        for opa, opb in LAYOUTS.values():
            assert lib.b200_gemm_workspace_bytes_op(opa, opb, 0, n, k, mode) == 0
    assert lib.b200_gemm_workspace_bytes_op(2, 0, 64, 64, 64, 2) == 0


def test_workspace_bytes_op_counts_transposes_and_planes(gemm):
    """The sizes of the routes in the header's table: TF32 NT transposes nothing, TF32 TN holds B^T and A, STRICT
    holds each transposed operand, the split modes hold planes padded in the layout they are stored in."""
    ws = gemm.lib.b200_gemm_workspace_bytes_op
    r16 = lambda x, e: -(-x * e // 16) * 16 // e
    r1k = lambda b: -(-b // 1024) * 1024
    m, n, k = 200, 136, 264
    assert ws(OP_N, OP_T, m, n, k, F32_MODES["tf32"]) == 0
    assert ws(OP_T, OP_N, m, n, k, F32_MODES["tf32"]) == r1k(n * r16(k, 4) * 4) + m * r16(k, 4) * 4
    assert ws(OP_T, OP_T, m, n, k, F32_MODES["tf32"]) == m * r16(k, 4) * 4
    assert ws(OP_N, OP_T, m, n, k, F32_MODES["strict"]) == k * r16(n, 4) * 4
    assert ws(OP_T, OP_T, m, n, k, F32_MODES["strict"]) == r1k(m * r16(k, 4) * 4) + k * r16(n, 4) * 4
    p8, r32 = (lambda c: -(-c // 8) * 8), (lambda r: -(-r // 32) * 32)
    # BF16X3, TN: A^T planes k x m stacked with zero rows to round32(k), B planes as for NN
    assert ws(OP_T, OP_N, m, n, k, F32_MODES["bf16x3"]) == r1k(3 * r32(k) * p8(m) * 2) + 3 * r32(k) * p8(n) * 2
    # BF16X2, NT: B^T planes n x k
    assert ws(OP_N, OP_T, m, n, k, F32_MODES["bf16x2"]) == r1k(2 * m * p8(k) * 2) + 2 * n * p8(k) * 2
    # F16X2, NT: planes of A and B^T, then A's and B^T's row maxima
    a, b = 2 * m * p8(k) * 2, 2 * n * p8(k) * 2
    assert ws(OP_N, OP_T, m, n, k, F32_MODES["f16x2"]) == r1k(r1k(r1k(a) + b) + 4 * m) + 4 * n


def test_workspace_bytes_nn_is_what_the_route_reserves(gemm):
    """NN: an explicit mode gives exactly what its route reserves, AUTO the largest of the routes it may take."""
    ws = gemm.lib.b200_gemm_workspace_bytes
    r1k = lambda b: -(-b // 1024) * 1024
    p8, r32 = (lambda c: -(-c // 8) * 8), (lambda r: -(-r // 32) * 32)
    m, n, k = 200, 136, 264
    assert ws(m, n, k, F32_MODES["strict"]) == 0
    assert ws(m, n, k, F32_MODES["tf32"]) == n * -(-k // 4) * 4 * 4                     # B^T, 16-byte pitch
    for mode, np_ in (("bf16x3", 3), ("bf16x2", 2)):
        assert ws(m, n, k, F32_MODES[mode]) == r1k(np_ * m * p8(k) * 2) + np_ * r32(k) * p8(n) * 2
    # F16X2: planes of A and B, then A's row maxima
    assert ws(m, n, k, F32_MODES["f16x2"]) == r1k(r1k(2 * m * p8(k) * 2) + 2 * r32(k) * p8(n) * 2) + 4 * m
    # AUTO at m*n*k = 1.28e9 with the default F16X2 (or BF16X3) takes BF16X3, whose planes hold 960,000,000 bytes
    if gemm.lib.b200_gemm_default_f32_mode() in (F32_MODES["f16x2"], F32_MODES["bf16x3"]):
        assert ws(16, 16, 5_000_000, F32_MODES["auto"]) >= 960_000_000


# ==== the Python layout resolver (no GPU) =====================================================================
def test_operand_layout_resolver(gemm):
    lay = gemm.operand_layout
    assert lay((6, 10), (10, 1)) == (OP_N, 10)                      # row-major
    assert lay((10, 6), (1, 10)) == (OP_T, 10)                      # x.T: stored 6 x 10
    assert lay((6, 7), (10, 1)) == (OP_N, 10)                       # x[:, :7]: ld > cols
    assert lay((7, 6), (1, 10)) == (OP_T, 10)                       # x[:, :7].T
    assert lay((3, 6), (20, 1)) == (OP_N, 20)                       # every other row
    assert lay((1, 10), (10, 1)) == (OP_N, 10) and lay((1, 10), (999, 1)) == (OP_N, 999)
    assert lay((6, 1), (1, 1)) == (OP_N, 1) and lay((6, 1), (10, 1)) == (OP_N, 10)   # a single column
    assert lay((1, 6), (1, 10)) == (OP_T, 10)                       # one row of a transposed view
    for shape, strides in (((6, 10), (10, 2)), ((6, 10), (2, 12)), ((10, 6), (2, 20)), ((4, 4), (0, 0))):
        with pytest.raises(ValueError):
            lay(shape, strides)
    if torch is not None:                                           # the same on real (CPU) tensors
        W = torch.zeros((12, 20))
        for t, want in ((W, (OP_N, 20)), (W.t(), (OP_T, 20)), (W[:, :7], (OP_N, 20)), (W[:, :7].t(), (OP_T, 20)),
                        (W[2:5, 3:11].t(), (OP_T, 20))):
            assert lay(tuple(t.shape), t.stride()) == want
        with pytest.raises(ValueError):
            lay(tuple(W[:, ::2].shape), W[:, ::2].stride())


# ==== GPU helpers ===============================================================================================
@pytest.fixture
def hooks(gemm):
    lib = gemm.lib
    try:
        yield lib
    finally:
        lib.b200_gemm_debug_set_bn(0)
        lib.b200_gemm_debug_set_split_tail(1)
        lib.b200_gemm_debug_set_group_rows(0)
        lib.b200_gemm_debug_set_ffma_variant(-1)
        lib.b200_gemm_debug_set_split_chunk(-1, -1)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stored(X, aligned):
    """X (rows x cols) as a row-major device view: aligned = 16-element pitch and 16-byte base (TMA-able);
    otherwise pitch cols + 1 and a base one element past an allocation (no operand type can use TMA)."""
    r, c = X.shape
    if aligned:
        buf = torch.zeros((r, ts.pitch(c)), dtype=X.dtype, device="cuda")
        v = buf[:, :c]
    else:
        flat = torch.zeros(r * (c + 1) + 1, dtype=X.dtype, device="cuda")
        v = flat.as_strided((r, c), (c + 1, 1), 1)
    v.copy_(X)
    return v


def operand(X, op, aligned):
    """(view passed to the library, ld): op = N stores X, op = T stores X^T."""
    v = stored(X.t() if op == OP_T else X, aligned)
    return v, v.stride(0)


OUT_DT = {"bf16": "float32", "bf16_obf16": "bfloat16", "s8": "int32"}


def out_buf(kind, m, n):
    dt = getattr(torch, OUT_DT.get(kind, "float32"))
    buf = torch.empty((m, n + 1 + n % 2), dtype=dt, device="cuda")
    buf.fill_(float("nan") if dt.is_floating_point else 77)
    return buf


def call(gemm, kind, mode, op_a, op_b, A, lda, B, ldb, buf, n, alpha=1.0, beta=0.0):
    """One library call into buf[:, :n]; returns (launches issued, kernel name)."""
    lib = gemm.lib
    m = buf.shape[0]
    k = A.shape[1] if op_a == OP_N else A.shape[0]
    ldc = buf.stride(0)
    before = lib.b200_gemm_launch_count()
    if kind in ("bf16", "bf16_obf16"):
        rc = lib.b200_gemm_bf16_op(op_a, op_b, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, buf.data_ptr(), ldc,
                                   0 if kind == "bf16" else 1, None)
    elif kind == "s8":
        rc = lib.b200_gemm_s8s32_op(op_a, op_b, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, buf.data_ptr(), ldc, None)
    else:
        rc = lib.b200_gemm_f32_op(op_a, op_b, m, n, k, alpha, A.data_ptr(), lda, B.data_ptr(), ldb, beta, buf.data_ptr(),
                                  ldc, F32_MODES[mode], None)
    assert rc == 0, (kind, mode, rc)
    return lib.b200_gemm_launch_count() - before, gemm.last_kernel()


def bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def same_bits(x, y):
    if x.dtype.is_floating_point:
        nx, ny = torch.isnan(x), torch.isnan(y)
        return bool(torch.equal(nx, ny)) and bool(torch.equal(bits(x)[~nx], bits(y)[~ny]))
    return bool(torch.equal(x, y))


LAUNCHES = {   # per layout NN, NT, TN, TT on the tensor-core / FFMA routes (include/b200gemm.h)
    "bf16": (1, 1, 1, 1), "bf16_obf16": (1, 1, 1, 1), "tf32": (2, 1, 3, 2), "s8": (2, 1, 3, 2),
    "bf16x3": (2, 2, 2, 2), "bf16x2": (2, 2, 2, 2), "f16x2": (4, 3, 5, 4), "strict": (1, 2, 2, 3)}
LAY_INDEX = {"nn": 0, "nt": 1, "tn": 2, "tt": 3}
TC_NAME = {"bf16": "tc_bf16", "bf16_obf16": "tc_bf16_obf16", "tf32": "tc_tf32", "s8": "tc_s8",
           "bf16x3": "tc_bf16x3", "bf16x2": "tc_bf16x2", "f16x2": "tc_f16x2"}
GENERIC = {"bf16": "generic_bf16_64x64", "bf16_obf16": "generic_bf16_64x64", "s8": "generic_s8_64x64",
           "tf32": "generic_f32_64x64", "strict": "generic_f32_64x64"}


def expected_route(route, lay, bn, aligned, fat=False):
    """(launches, kernel name) of a call on `route` (a kind or a concrete fp32 mode)."""
    if not aligned and route in GENERIC:
        return 1, GENERIC[route]
    n = LAUNCHES[route][LAY_INDEX[lay]]
    if route == "strict":
        return n, "ffma_fat_128x256x32_tma" if fat else "ffma_128x128x32_tma"
    tag = "" if lay == "nn" or route in ("tf32", "s8") else "_" + lay     # tf32 / int8 run the NN instantiations
    return n, f"{TC_NAME[route]}{tag}_128x{bn}"


def make_logical(kind, m, n, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "s8":
        return (torch.randint(-127, 128, (m, k), device="cuda", generator=g, dtype=torch.int8),
                torch.randint(-127, 128, (k, n), device="cuda", generator=g, dtype=torch.int8))
    A = torch.rand((m, k), device="cuda", generator=g) * 2 - 1
    B = torch.rand((k, n), device="cuda", generator=g) * 2 - 1
    if kind in ("bf16", "bf16_obf16"):
        A, B = A.bfloat16(), B.bfloat16()
    return A, B


def check_ref(kind, route, A, B, got, alpha=1.0, beta=0.0, c0=None):
    t = alpha * (A.double() @ B.double())
    if c0 is not None and beta != 0.0:
        t = t + beta * c0.double()
    if kind == "s8":
        assert torch.equal(got.long(), t.long())
    elif kind == "bf16_obf16":
        c = got.double()
        assert bool(((c - t).abs() <= t.abs() * 2.0 ** -8 + ts.TOL["bf16"] * t.abs().max()).all())
    else:
        tol = ts.TOL_STRICT if route == "strict" else ts.TOL[route]
        err = float((got.double() - t).abs().max() / t.abs().max())
        assert err <= tol, (kind, route, err)


def compare_layouts(gemm, kind, mode, m, n, k, seed, aligned=True, alpha=1.0, beta=0.0, route=None, bn=None, fat=False,
                    layouts=("nt", "tn", "tt"), A=None, B=None, reference=True):
    """Every layout against NN on row-major copies (same alignment class): bits, route, reference."""
    if A is None:
        A, B = make_logical(kind, m, n, k, seed)
    route = route or (mode if kind == "f32" else kind)
    c0 = torch.rand((m, n), device="cuda") * 2 - 1 if beta != 0.0 else None
    results = {}
    for lay in ("nn",) + tuple(layouts):
        op_a, op_b = (OP_N, OP_N) if lay == "nn" else LAYOUTS[lay]
        Av, lda = operand(A, op_a, aligned)
        Bv, ldb = operand(B, op_b, aligned)
        buf = out_buf(kind, m, n)
        if c0 is not None:
            buf[:, :n] = c0
        launches, name = call(gemm, kind, mode, op_a, op_b, Av, lda, Bv, ldb, buf, n, alpha, beta)
        if bn is not None:
            assert (launches, name) == expected_route(route, lay, bn, aligned, fat), (kind, mode, lay, launches, name)
        results[lay] = (buf, name)
    base = results["nn"][0]
    for lay in layouts:
        assert same_bits(results[lay][0], base), (kind, mode, lay, (m, n, k), aligned, results[lay][1])
    if reference:
        check_ref(kind, route, A, B, base[:, :n], alpha, beta, c0)
    pad = base[:, n:]
    assert bool(torch.isnan(pad).all()) if pad.dtype.is_floating_point else bool((pad == 77).all())
    return results


# ==== bit identity with NN, routes and the float64 reference: the wgmma kinds =====================================
TC_KINDS = ("bf16", "bf16_obf16", "tf32", "s8", "bf16x3", "bf16x2", "f16x2")


def shapes_for(kind, sms):
    """Forced tile widths with M / N / K tails and ld > dim, and one K-split tail shape.  (m, n, k, bn)"""
    sk = {"bf16x3": "bf16x3", "bf16x2": "bf16x2", "f16x2": "f16x2"}.get(kind, kind)
    out = [c for c in ts.width_cases(sk) if (c[0], c[1] - c[3]) in ((1, -8), (129, 8), (389, c[3] + 8))]
    if kind in ts.SPLIT_KINDS:
        out.append(ts.split_case(kind, 2, sms, False))
    return out


@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
@pytest.mark.parametrize("kind", TC_KINDS)
def test_bit_identical_to_nn(gemm, hooks, sms, kind, aligned):
    f32_kind = kind in ("tf32", "bf16x3", "bf16x2", "f16x2")
    for i, (m, n, k, bn) in enumerate(shapes_for(kind, sms)):
        hooks.b200_gemm_debug_set_bn(bn)
        compare_layouts(gemm, "f32" if f32_kind else kind, kind if f32_kind else None, m, n, k, 10 + i, aligned,
                        route=kind, bn=bn)


@gpu
@pytest.mark.parametrize("alpha,beta", [(1.0, 1.0), (-0.75, 0.5), (2.0 ** -70, 2.0 ** 70)])
@pytest.mark.parametrize("mode", ["strict", "tf32", "bf16x3", "bf16x2", "f16x2"])
def test_alpha_beta_bit_identical_to_nn(gemm, hooks, sms, mode, alpha, beta):
    """C = alpha op(A) op(B) + beta C, and C += op(A) op(B), with a K-split tail on the tensor-core modes."""
    m, n, k, bn = ts.split_case(mode if mode != "strict" else "tf32", 2, sms, False)
    for aligned in (True, False):
        compare_layouts(gemm, "f32", mode, m, n, k, 40, aligned, alpha=alpha, beta=beta)


@gpu
@pytest.mark.parametrize("fat", [False, True], ids=["128x128", "fat_128x256"])
def test_strict_routes(gemm, oracle, hooks, sms, fat):
    """STRICT on TMA-able operands: transposes into the workspace, then the unchanged FFMA kernel (half tiles in
    the last round); bit-exact against the oracle as well as against NN.  Unaligned operands: the generic kernel
    reading the operands with their strides."""
    m, n, k = ts.strict_case(sms, fat)
    hooks.b200_gemm_debug_set_ffma_variant((2 if fat else 0) | 1)
    for aligned, shape in ((True, (m, n, k)), (False, (200, 136, 100))):
        A, B = make_logical("f32", *shape, 50)
        res = compare_layouts(gemm, "f32", "strict", *shape, 50, aligned, bn=0, fat=fat, A=A, B=B)
        want = _libs.ref_f32_fma(oracle, A.cpu().numpy(), B.cpu().numpy())
        assert np.array_equal(res["nn"][0][:, :shape[1]].cpu().numpy(), want)


AUTO_CASES = {"strict": (256, 256, 256), "bf16x3": (1024, 1024, 640), "f16x2": (1152, 1152, 1024)}


@gpu
@pytest.mark.parametrize("route", list(AUTO_CASES))
def test_auto_routes(gemm, hooks, route):
    if gemm.lib.b200_gemm_default_f32_mode() != gemm.F32_F16X2:
        pytest.skip("the default fp32 mode was changed in the environment")
    m, n, k = AUTO_CASES[route]
    compare_layouts(gemm, "f32", "auto", m, n, k, 60, True, route=route, bn=128)


# ==== range edges and known answers of the split modes ===========================================================
@gpu
@pytest.mark.parametrize("mode", fr.SPLIT_MODES)
def test_full_range_bit_identical_to_nn(gemm, hooks, mode):
    """Subnormal maxima, FLT_MAX, an unscale of 2^256, inf and NaN: the pre-pass role swap keeps every bit."""
    A, B = fr.range_operands(256, 256, 256, 42)
    for aligned in (True, False):
        compare_layouts(gemm, "f32", mode, 256, 256, 256, 0, aligned, A=fr.dev(A), B=fr.dev(B), reference=False,
                        route=mode, bn=128)


@gpu
@pytest.mark.parametrize("lay", list(LAYOUTS))
@pytest.mark.parametrize("mode", fr.SPLIT_MODES)
def test_known_answer_bit_exact(gemm, hooks, mode, lay):
    A, B, _ = fr.ka_case(mode, "plain")
    m, n = A.shape[0], B.shape[1]
    op_a, op_b = LAYOUTS[lay]
    Av, lda = operand(fr.dev(A), op_a, True)
    Bv, ldb = operand(fr.dev(B), op_b, True)
    buf = out_buf("f32", m, n)
    call(gemm, "f32", mode, op_a, op_b, Av, lda, Bv, ldb, buf, n)
    assert gemm.last_kernel() == f"{TC_NAME[mode]}_{lay}_128x128"
    got = buf[:, :n].cpu().numpy()
    want = fr.f32(fm.model(A, B, mode))
    bad = fm.bits(got) != fm.bits(want)
    assert not bad.any(), int(bad.sum())


# ==== the tensor-level interface =====================================================================================
@gpu
def test_python_gemm_reads_transposed_views_in_place(gemm):
    g = torch.Generator(device="cuda").manual_seed(70)
    x = torch.rand((300, 520), device="cuda", generator=g) * 2 - 1
    W = torch.rand((264, 520), device="cuda", generator=g) * 2 - 1          # n x k, as a linear layer holds it
    assert same_bits(gemm.gemm(x, W.t()), gemm.gemm_f32(x, W.t().contiguous()))      # AUTO
    want = gemm.gemm_f32(x, W.t().contiguous(), mode=gemm.F32_F16X2)
    out = torch.empty((300, 264), device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    gemm.gemm(x, W.t(), out=out, mode=gemm.F32_F16X2)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() == before                      # no copy of W was made
    assert gemm.last_kernel() == "tc_f16x2_nt_128x128"
    assert same_bits(out, want)
    # A transposed, a sliced view with ld > dim, bf16 and int8
    xt = torch.rand((520, 304), device="cuda", generator=g)[:, :300].t()     # ld 304: TMA-able, like the copy's
    assert same_bits(gemm.gemm(xt, W.t(), mode=gemm.F32_TF32), gemm.gemm_f32(xt.contiguous(), W.t().contiguous(), mode=gemm.F32_TF32))
    xb, Wb = x.bfloat16(), W.bfloat16()
    assert same_bits(gemm.gemm(xb, Wb.t(), out_dtype=torch.bfloat16), gemm.gemm_bf16(xb, Wb.t().contiguous(), out_dtype=torch.bfloat16))
    x8 = torch.randint(-127, 128, (300, 520), device="cuda", generator=g, dtype=torch.int8)
    W8 = torch.randint(-127, 128, (264, 520), device="cuda", generator=g, dtype=torch.int8)
    before = gemm.launch_count()
    got = gemm.gemm(x8, W8.t())
    assert gemm.launch_count() - before == 1                                # B^T is the K-major operand: no transpose
    assert torch.equal(got, gemm.gemm_s8s32(x8, W8.t().contiguous()))
    c0 = torch.rand((300, 264), device="cuda", generator=g)
    o1, o2 = c0.clone(), c0.clone()
    gemm.gemm(x, W.t(), out=o1, alpha=0.5, beta=-2.0, mode=gemm.F32_BF16X3)
    gemm.gemm_f32_ex(0.5, x, W.t().contiguous(), -2.0, o2, mode=gemm.F32_BF16X3)
    assert same_bits(o1, o2)
    with pytest.raises(ValueError):
        gemm.gemm(x, torch.rand((520, 528), device="cuda")[:, ::2])             # neither layout
