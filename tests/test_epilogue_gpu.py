"""Bias vector and ReLU / GELU fused into the epilogue of the 16-bit GEMMs: b200_gemm_bf16_epi, b200_gemm_f16_epi.

Per element the library computes, in fp32, t = fma(beta, float(C), alpha * x), t = t + float(bias[j]), y = act(t) and
stores round_out(y) (include/b200gemm.h).  The tests pin each step:
- the activation on every finite 16-bit value (A = I, so t is B), bit for bit for ReLU, within a derived bound of the
  float64 function for the GELUs, and bit-identical between the tensor-core and the generic route;
- the bias add bit for bit against a numpy float32 model on dyadic operands (an exact accumulator);
- 16-bit C as the round-to-nearest-even rounding of fp32 C;
- no K-split tail, the layouts, the zero rules and the identity case (null bias, B200_ACT_NONE = the _ex call).
Shapes, routes and helpers come from test_f16_gemm_gpu.py and the schedule model of test_tile_schedules_gpu.py.
Output buffers start as NaN and whole buffers, padding included, are compared.

The argument checks, the Python refusals and the schedule model need no GPU."""
import ctypes as C

import numpy as np
import pytest

import test_f16_gemm_gpu as f16
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
ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3
ACTS = {"none": ACT_NONE, "relu": ACT_RELU, "gelu": ACT_GELU, "gelu_tanh": ACT_GELU_TANH}
LAYS, OPS, KINDS16 = f16.LAYS, f16.OPS, f16.KINDS16
GENERIC = f16.GENERIC


# ==== schedule model (no GPU) ====================================================================================
# launch_tc in csrc/capi.cu: an epilogue kernel never takes the K-split tail (the activation must see the complete
# sum), whatever the C type; its tile widths are those of the plain 16-bit kernels (pick_bn(m, n, true)).
def epi_split(m, n, k, kind, bn, sms):
    """kind: a KINDS16 kind (fp16 runs bf16's schedule) or a kind of the schedule model."""
    kind = KINDS16[kind][4] if kind in KINDS16 else kind
    return ts.tc_split(m, n, k, kind, bn, sms, split_tail=False)


def epi_name(kind, lay, bn):
    """The epilogue kernel of a KINDS16 kind: "_epi" after the C-type part, then the layout."""
    return f"{KINDS16[kind][3]}_epi{'' if lay == 'nn' else '_' + lay}_128x{bn}"


@pytest.mark.parametrize("sms", [132, 114])
def test_epilogue_never_splits(sms):
    """On a 132-SM H100 SXM and a 114-SM H100 PCIe: every shape whose plain fp32-C call splits 2, 3 or 4 ways (with
    and without full rounds before the tail) runs whole tiles under the epilogue, at the same tile width."""
    for split in (2, 3, 4):
        for rounds in (False, True):
            m, n, k, bn = ts.split_case("bf16", split, sms, rounds)
            assert ts.tc_split(m, n, k, "bf16", bn, sms) == split
            assert ts.pick_bn(m, n, sms, "bf16", force=bn) == bn
            for kind in KINDS16:
                assert epi_split(m, n, k, kind, bn, sms) == 1
    for m, n, k, bn in ts.width_cases("bf16"):
        assert epi_split(m, n, k, "bf16", bn, sms) == 1
    assert epi_name("f16", "tn", 192) == "tc_f16_epi_tn_128x192"
    assert epi_name("bf16_obf16", "nn", 256) == "tc_bf16_obf16_epi_128x256"


# ==== argument checks (no GPU: every case returns before the device is touched) ===================================
def test_epi_argument_validation(gemm):
    lib = gemm.lib
    buf = (C.c_float * 256)()
    m, n, k = 4, 6, 8

    def call(fn, ot, act, mm=m, nn=n, a=buf, lda=k, ldb=n, c=buf, ldc=n, bias=buf, opa=OP_N, opb=OP_N, al=0.5):
        return fn(opa, opb, mm, nn, k, al, a, lda, buf, ldb, 0.25, c, ldc, ot, bias, act, None)

    for fn, ot16, bad16 in ((lib.b200_gemm_bf16_epi, OUT_BF16, OUT_F16), (lib.b200_gemm_f16_epi, OUT_F16, OUT_BF16)):
        for act in (-1, 4, 7, 1 << 20):                                  # a bad act, even on an empty problem
            assert call(fn, OUT_F32, act) == -1 and call(fn, OUT_F32, act, mm=0) == -1, act
            assert call(fn, OUT_F32, act, bias=None) == -1, act
        for act in ACTS.values():
            for bias in (buf, None):
                if bias is None and act == ACT_NONE:
                    continue                                             # the _ex call: its own tests
                for ot in (bad16, 3, -1):                                # out_type pairing
                    assert call(fn, ot, act, bias=bias) == -1, (ot, act)
                assert call(fn, ot16, act, bias=bias, a=None) == -1       # null A
                assert call(fn, ot16, act, bias=bias, c=None) == -1       # null C
                assert call(fn, ot16, act, bias=bias, lda=k - 1) == -1    # ld below its op's minimum
                assert call(fn, ot16, act, bias=bias, ldb=n - 1) == -1
                assert call(fn, ot16, act, bias=bias, ldc=n - 1) == -1
                assert call(fn, ot16, act, bias=bias, opa=OP_T, lda=m - 1) == -1
                assert call(fn, ot16, act, bias=bias, opb=OP_T, ldb=k - 1) == -1
                assert call(fn, ot16, act, bias=bias, opa=2) == -1        # a bad op
                assert call(fn, ot16, act, bias=bias, mm=-1) == -1
                # empty problems are no-ops, null bias and null pointers included
                assert fn(OP_T, OP_N, 0, n, k, 0.5, None, 1, None, 1, 2.0, None, 1, ot16, None, act, None) == 0
                assert fn(OP_N, OP_T, m, 0, k, 1.0, None, 1, None, 1, 0.0, None, 1, OUT_F32, None, act, None) == 0
                assert call(fn, OUT_F32, act, bias=bias, mm=0) == 0


def test_python_epilogue_refusals(gemm):
    """Refused before anything touches a device: fp32 / int8 operands (TypeError), a bias of another dtype or length,
    a 2-D bias or an unknown activation (ValueError)."""
    if torch is None:
        pytest.skip("needs torch")
    x16, w16 = torch.zeros((4, 8), dtype=torch.float16), torch.zeros((8, 6), dtype=torch.float16)
    for dt in (torch.float32, torch.int8):
        x, w = torch.zeros((4, 8), dtype=dt), torch.zeros((8, 6), dtype=dt)
        with pytest.raises(TypeError):
            gemm.gemm(x, w, activation="relu")
        with pytest.raises(TypeError):
            gemm.gemm(x, w, bias=torch.zeros(6, dtype=dt))
    with pytest.raises(TypeError):
        gemm.gemm(x16, w16.bfloat16(), activation="gelu")                # mixed operand dtypes
    for dt in (torch.float16, torch.bfloat16):
        x, w = x16.to(dt), w16.to(dt)
        other = torch.bfloat16 if dt == torch.float16 else torch.float16
        for bad in (torch.zeros(6, dtype=other), torch.zeros(6, dtype=torch.float32), torch.zeros(5, dtype=dt),
                    torch.zeros(7, dtype=dt), torch.zeros((1, 6), dtype=dt)):
            with pytest.raises(ValueError):
                gemm.gemm(x, w, bias=bad)
        for bad in ("silu", "GELU", "tanh", 1):
            with pytest.raises(ValueError):
                gemm.gemm(x, w, activation=bad)


# ==== GPU helpers ==================================================================================================
def dt(name):
    return getattr(torch, name)


def call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, k, bias, act, alpha=1.0, beta=0.0):
    """One b200_gemm_*_epi call into buf[:, :n]; returns (launches issued, kernel name).  bias: a tensor (its
    data_ptr is passed as is, so a view at an odd element offset tests a 2-byte-aligned bias) or None."""
    lib = gemm.lib
    ind, _, ot, _, _ = KINDS16[kind]
    fn = lib.b200_gemm_f16_epi if ind == "float16" else lib.b200_gemm_bf16_epi
    m, ldc = buf.shape[0], buf.stride(0)
    a, b = (Av.data_ptr() if Av is not None else None), (Bv.data_ptr() if Bv is not None else None)
    before = lib.b200_gemm_launch_count()
    rc = fn(op_a, op_b, m, n, k, alpha, a, lda, b, ldb, beta, buf.data_ptr(), ldc, ot,
            bias.data_ptr() if bias is not None else None, act, None)
    assert rc == 0, (kind, rc)
    return lib.b200_gemm_launch_count() - before, gemm.last_kernel()


def epi_route(kind, lay, bn, aligned):
    return (1, GENERIC[KINDS16[kind][0]]) if not aligned else (1, epi_name(kind, lay, bn))


def run_epi(gemm, kind, A, B, aligned, bias, act, bn=None, alpha=1.0, beta=0.0, c0=None, lays=LAYS):
    """Each layout on operands stored as op requires; asserts the route and the untouched padding, returns
    {layout: buf}."""
    m, k = A.shape
    n = B.shape[1]
    res = {}
    for lay in lays:
        op_a, op_b = OPS[lay]
        Av, lda = tr.operand(A, op_a, aligned)
        Bv, ldb = tr.operand(B, op_b, aligned)
        buf = f16.out_buf16(kind, m, n, c0)
        got = call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, k, bias, act, alpha, beta)
        if bn is not None:
            assert got == epi_route(kind, lay, bn, aligned), (kind, lay, got)
        else:
            assert got[0] == 1 and (got[1] == GENERIC[KINDS16[kind][0]]) == (not aligned), (kind, lay, got)
        assert bool(torch.isnan(buf[:, n:]).all()), (kind, lay)
        res[lay] = buf
    return res


def bias_vec(ind, n, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(n, device="cuda", generator=g) * (hi - lo) + lo).to(dt(ind))


def odd_view(v):
    """v at a 2-byte (not 4-byte) aligned address: one element into a fresh allocation."""
    buf = torch.zeros(v.numel() + 1, dtype=v.dtype, device="cuda")
    out = buf[1:]
    out.copy_(v)
    assert out.data_ptr() % 4 == 2
    return out


def model_f32(x, bias, alpha=1.0, beta=0.0, c0=None, act="none"):
    """The numpy float32 model fl(fma(beta, C, alpha * x) + b), then ReLU, of an exact accumulator x (float64 array
    exactly representable in fp32); alpha * x, beta * C and their sum are exact for the dyadic cases it is used on."""
    x32 = x.astype(np.float32)
    t = (np.float64(alpha) * x32.astype(np.float64))
    if c0 is not None and beta != 0.0:
        t = t + np.float64(beta) * c0.astype(np.float64)
    t32 = t.astype(np.float32)
    assert np.array_equal(t32.astype(np.float64), t), "the model case is not exact"
    y = t32 + bias.astype(np.float32)[None, :] if bias is not None else t32
    if act == "relu":
        y = np.where(y < 0, np.float32(0), y).astype(np.float32)
    return y


def np_of(t):
    return t.detach().float().cpu().numpy()


def same_np(got, want):
    g, w = np_of(got), np.asarray(want, np.float32)
    ng, nw = np.isnan(g), np.isnan(w)
    return bool(np.array_equal(ng, nw)) and bool(np.array_equal(g[~ng].view(np.int32), w[~nw].view(np.int32)))


# ==== 1. the activation on every finite 16-bit value ================================================================
def all_finite(ind):
    """Every finite bit pattern of the type, as a 256 x n matrix (n = 255 for bf16, 248 for fp16)."""
    bits = torch.arange(0, 1 << 16, dtype=torch.int32)
    v = bits.to(torch.int16).view(dt(ind))
    v = v[torch.isfinite(v.float())]
    assert v.numel() % 256 == 0
    return v.view(256, -1).cuda()


def gelu64(t, act):
    """The float64 function on t (finite)."""
    if act == "gelu":
        return 0.5 * t * torch.special.erfc(-t / np.sqrt(2.0))
    return 0.5 * t * (1.0 + torch.tanh(np.sqrt(2.0 / np.pi) * (t + 0.044715 * t ** 3)))


GELU_BOUND = (2.0 ** -19, 2.0 ** -22, 2.0 ** -149)


@gpu
@pytest.mark.parametrize("ind", ["float16", "bfloat16"])
def test_activation_table_exhaustive(gemm, ind):
    """A = I (256 x 256), B = every finite value of the 16-bit type: t is B (up to the sign of zero), read back from
    the B200_ACT_NONE call with a -0 bias (t + -0 is t).  fp32 C:
    - ReLU equals where(t < 0, +0, t) bit for bit;
    - GELU and GELU_TANH lie within 2^-19 |g(t)| + 2^-22 |t| + 2^-149 of the float64 function g.  Derivation, with
      the CUDA Math API maxima (erfcf 4 ulp, tanhf 2 ulp) and u = 2^-24:
      GELU = fl(fl(0.5 t) * erfcf(fl(-t / sqrt 2))).  For t >= 0, erfc(z) lies in [1, 2] and changes slowly, so the
      argument's rounding (2u) costs under u relative; with erfcf's 4 ulp (<= 8u) and the final product (u) the
      result is within about 10u < 2^-19 relative.  For t < 0 the argument's rounding is amplified by
      z erfc'(z) / erfc(z) ~ 2 z^2 = t^2, an absolute error of about |g| t^2 2u = |t| Phi(t) |t| 2u <= |t| 2^-25
      (|t| Phi(t) <= 0.25), inside 2^-22 |t|.  0.5 t is exact unless t is subnormal, and any product that lands in
      the subnormal range rounds by at most 2^-150: the 2^-149 term.
      GELU_TANH = fl(fl(0.5 t) * fl(1 + tanhf(u(t)))), u(t) computed with 5 roundings (<= 6u relative).  The error of
      1 + tanh is absolute: tanhf's 2 ulp (<= 2^-23 for |tanh| in [0.5, 1)) plus sech^2(u) |u| 6u <= 0.45 * 6u,
      together under 2^-22; times 0.5 |t| that is inside 2^-22 |t|.  For t >= 0, 1 + tanh >= 1 and the same absolute
      error is a relative one under 2^-19.
    - Tensor-core and generic route give the same bits.
    - +inf, -inf and NaN reach the activation through the bias (t = x + inf): +inf, -0 (GELUs) / +0 (ReLU) and NaN,
      in their column only."""
    A = torch.eye(256, device="cuda").to(dt(ind))
    B = all_finite(ind)
    n = B.shape[1]
    kind = "f16" if ind == "float16" else "bf16"
    mz = torch.full((n,), -0.0, device="cuda").to(dt(ind))
    t = {al: run_epi(gemm, kind, A, B, al, mz, ACT_NONE, lays=("nn",))["nn"][:, :n] for al in (True, False)}
    assert tr.same_bits(t[True], t[False])
    t = t[True]
    nz = B.float() != 0
    assert tr.same_bits(t[nz], B.float()[nz]) and bool((t[~nz] == 0).all())
    t64 = t.double()
    for act in ("relu", "gelu", "gelu_tanh"):
        res = {al: run_epi(gemm, kind, A, B, al, mz, ACTS[act], lays=("nn",))["nn"][:, :n] for al in (True, False)}
        assert tr.same_bits(res[True], res[False]), act
        y = res[True]
        if act == "relu":
            assert tr.same_bits(y, torch.where(t < 0, torch.zeros_like(t), t))
        else:
            g = gelu64(t64, act)
            r, a, s = GELU_BOUND
            err = (y.double() - g).abs() - (r * g.abs() + a * t64.abs() + s)
            assert bool(torch.isfinite(y).all()) and float(err.max()) <= 0, (act, float(err.max()))
            assert tr.same_bits(y[t == 0], t[t == 0] * 0.5)      # gelu(+-0) = +-0
    # non-finite t through the bias: columns 3, 50 and 100 get +inf, -inf and NaN
    bias = mz.clone()
    bias[3], bias[50], bias[100] = float("inf"), float("-inf"), float("nan")
    spec = torch.zeros(n, dtype=torch.bool, device="cuda")
    spec[[3, 50, 100]] = True
    for act in ACTS:
        for al in (True, False):
            y = run_epi(gemm, kind, A, B, al, bias, ACTS[act], lays=("nn",))["nn"][:, :n]
            want_ninf = {"none": float("-inf"), "relu": 0.0, "gelu": -0.0, "gelu_tanh": -0.0}[act]
            assert bool((y[:, 3] == float("inf")).all()), (act, al)
            assert tr.same_bits(y[:, 50], torch.full((256,), want_ninf, device="cuda")), (act, al)
            assert bool(torch.isnan(y[:, 100]).all()), (act, al)
            assert bool(torch.isfinite(y[:, ~spec]).all()), (act, al)


# ==== 2. the bias, bit-exact =========================================================================================
@gpu
@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("kind", ["bf16", "f16"])
def test_bias_known_answers(gemm, hooks, sms, kind, act):
    """Dyadic operands (an exact accumulator x) and C: fp32 C equals the numpy float32 model fl(fma(beta, C, alpha x)
    + b) (then ReLU) bit for bit, in every layout and forced width with M / N / K tails, for (1, 0) and a general
    (alpha, beta); a bias at a 2-byte (not 4-byte) aligned address gives the same bits."""
    ind = KINDS16[kind][0]
    for i, (m, n, k, bn) in enumerate(f16.shapes16(sms, ())):
        hooks.b200_gemm_debug_set_bn(bn)
        A, B = f16.logical16(kind, m, n, k, 1000 + i, dyadic=True)
        x = (A.double() @ B.double()).cpu().numpy()
        g = torch.Generator(device="cuda").manual_seed(1100 + i)
        c0 = torch.randint(-8, 9, (m, n), device="cuda", generator=g).float() / 8
        bias = bias_vec(ind, n, 1200 + i, -4.0, 4.0)
        bnp = np_of(bias)
        for alpha, beta in ((1.0, 0.0), (-0.75, 0.5)):
            want = model_f32(x, bnp, alpha, beta, np_of(c0), act)
            for bv in (bias, odd_view(bias)):
                for lay, buf in run_epi(gemm, kind, A, B, True, bv, ACTS[act], bn, alpha, beta, c0).items():
                    assert same_np(buf[:, :n], want), (kind, act, lay, (m, n, k, bn), alpha, beta)


# ==== 3. 16-bit C is the rounding of fp32 C ============================================================================
@gpu
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-0.75, 0.5), (3000.0, 0.5)], ids=["plain", "general", "overflow"])
@pytest.mark.parametrize("ind", ["float16", "bfloat16"])
def test_16bit_c_is_rounded_fp32_c(gemm, hooks, sms, ind, alpha, beta):
    """Under the same bias, activation and (alpha, beta), with fp32 C seeded with float(C16) and the split tail off
    for neither (the epilogue never splits), 16-bit C is the RNE rounding of fp32 C on both routes and in every
    layout; alpha = 3000 drives fp16 C past 65504 to +-inf."""
    k32, k16 = ("f16", "f16_of16") if ind == "float16" else ("bf16", "bf16_obf16")
    m, n, k, bn = ts.split_case("bf16", 2, sms, False)
    hooks.b200_gemm_debug_set_bn(bn)
    A, B = f16.logical16(k32, m, n, k, 1300)
    g = torch.Generator(device="cuda").manual_seed(1301)
    c16 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(dt(ind))
    bias = bias_vec(ind, n, 1302, -2.0, 2.0)
    overflowed = False
    for act in ACTS.values():
        for aligned in (True, False):
            r32 = run_epi(gemm, k32, A, B, aligned, bias, act, bn, alpha, beta, c16.float())
            r16 = run_epi(gemm, k16, A, B, aligned, bias, act, bn, alpha, beta, c16)
            for lay in LAYS:
                assert tr.same_bits(r16[lay][:, :n], r32[lay][:, :n].to(dt(ind))), (ind, act, lay, aligned)
            overflowed |= bool(torch.isinf(r16["nn"][:, :n]).any())
    assert overflowed == (ind == "float16" and alpha > 65504 / 100)


# ==== 4. no K-split tail ============================================================================================
@gpu
@pytest.mark.parametrize("split", [2, 3, 4])
@pytest.mark.parametrize("kind", ["bf16", "f16"])
def test_no_split_tail(gemm, hooks, sms, kind, split):
    """A shape whose plain fp32-C call splits the last round `split` ways: the epilogue call is one launch of the _epi
    kernel and bit-identical to the model applied to the plain call made with the split tail off."""
    m, n, k, bn = ts.split_case("bf16", split, sms, False)
    assert ts.tc_split(m, n, k, "bf16", bn, sms) == split and epi_split(m, n, k, kind, bn, sms) == 1
    hooks.b200_gemm_debug_set_bn(bn)
    ind = KINDS16[kind][0]
    A, B = f16.logical16(kind, m, n, k, 1400 + split)
    bias = bias_vec(ind, n, 1410 + split)
    Av, lda = tr.operand(A, OP_N, True)
    Bv, ldb = tr.operand(B, OP_N, True)
    split_buf = f16.out_buf16(kind, m, n)
    f16.call16(gemm, kind, OP_N, OP_N, Av, lda, Bv, ldb, split_buf, n, k)
    hooks.b200_gemm_debug_set_split_tail(0)
    plain = f16.out_buf16(kind, m, n)
    f16.call16(gemm, kind, OP_N, OP_N, Av, lda, Bv, ldb, plain, n, k)
    hooks.b200_gemm_debug_set_split_tail(1)
    x = np_of(plain[:, :n]).astype(np.float64)
    for act in ("none", "relu"):
        res = run_epi(gemm, kind, A, B, True, bias, ACTS[act], bn, lays=("nn",))["nn"]
        assert same_np(res[:, :n], model_f32(x, np_of(bias), act=act)), (kind, split, act)


# ==== 5. layouts ====================================================================================================
@gpu
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "ld_plus_1"])
@pytest.mark.parametrize("kind", list(KINDS16))
def test_layouts_bit_identical_to_nn(gemm, hooks, sms, kind, aligned):
    """NT / TN / TT equal NN bit for bit under a bias and each activation, with the route and kernel name of every
    forced width; the odd-address bias too."""
    ind = KINDS16[kind][0]
    for i, (m, n, k, bn) in enumerate(f16.shapes16(sms, ())):
        hooks.b200_gemm_debug_set_bn(bn)
        A, B = f16.logical16(kind, m, n, k, 1500 + i)
        bias = bias_vec(ind, n, 1550 + i)
        for act in ACTS.values():
            res = run_epi(gemm, kind, A, B, aligned, bias if i % 2 else odd_view(bias), act, bn, -0.75, 0.0)
            for lay in LAYS[1:]:
                assert tr.same_bits(res[lay], res["nn"]), (kind, lay, (m, n, k, bn), act, aligned)


# ==== 6. zero rules and the identity case ============================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_zero_rules(gemm, hooks, sms, kind):
    """alpha == 0 (NaN operands) and k == 0 store round(act(beta * float(C) + b)) in one pass; beta == 0 contributes +0
    and never reads C (NaN C leaves no trace).  fp32 C is checked against torch's fp32 ops (ReLU exactly; the GELUs
    against the library's own fp32-C result, rounded, for 16-bit C)."""
    m, n, k = 200, 136, 264
    ind, cdn = KINDS16[kind][0], KINDS16[kind][1]
    cd = dt(cdn)
    A, B = f16.logical16(kind, m, n, k, 1600)
    g = torch.Generator(device="cuda").manual_seed(1601)
    c0 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(cd)
    bias = bias_vec(ind, n, 1602)
    An, Bn = torch.full_like(A, float("nan")), torch.full_like(B, float("nan"))
    for aligned in (True, False):
        for lay in LAYS:
            op_a, op_b = OPS[lay]
            Av, lda = tr.operand(An, op_a, aligned)
            Bv, ldb = tr.operand(Bn, op_b, aligned)
            for act in ("none", "relu"):
                for beta in (0.5, 0.0):
                    t = (beta * c0.float() if beta != 0 else torch.zeros_like(c0.float())) + bias.float()[None, :]
                    want = (torch.relu(t) if act == "relu" else t).to(cd)
                    for kk, al in ((k, 0.0), (0, 1.0)):
                        buf = f16.out_buf16(kind, m, n, c0)
                        launches, _ = call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, buf, n, kk, bias, ACTS[act], al,
                                               beta)
                        assert launches == 1
                        assert tr.same_bits(buf[:, :n], want), (kind, lay, act, beta, kk)
                        assert bool(torch.isnan(buf[:, n:]).all())
            Av, lda = tr.operand(A, op_a, aligned)       # beta = 0: C is NaN and must not be read
            Bv, ldb = tr.operand(B, op_b, aligned)
            for act in ACTS.values():
                b_nan, b_zero = f16.out_buf16(kind, m, n), f16.out_buf16(kind, m, n, torch.zeros_like(c0))
                call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b_nan, n, k, bias, act, -0.75, 0.0)
                call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b_zero, n, k, bias, act, -0.75, 0.0)
                assert bool(torch.isfinite(b_nan[:, :n]).all()) and tr.same_bits(b_nan, b_zero), (kind, lay, act)


@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_null_bias_no_act_is_the_ex_call(gemm, hooks, sms, kind):
    """A null bias with B200_ACT_NONE: the bits, kernel name and launch count of b200_gemm_*_ex, for (1, 0) and a
    general (alpha, beta), the K-split tail of fp32 C included."""
    m, n, k, bn = ts.split_case("bf16", 2, sms, False)
    A, B = f16.logical16(kind, m, n, k, 1700)
    g = torch.Generator(device="cuda").manual_seed(1701)
    c0 = (torch.rand((m, n), device="cuda", generator=g) * 2 - 1).to(dt(KINDS16[kind][1]))
    for aligned in (True, False):
        for lay in LAYS:
            op_a, op_b = OPS[lay]
            Av, lda = tr.operand(A, op_a, aligned)
            Bv, ldb = tr.operand(B, op_b, aligned)
            for alpha, beta in ((1.0, 0.0), (-0.75, 0.5)):
                b1, b2 = f16.out_buf16(kind, m, n, c0), f16.out_buf16(kind, m, n, c0)
                r1 = f16.call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b1, n, k, alpha, beta)
                r2 = call_epi(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, b2, n, k, None, ACT_NONE, alpha, beta)
                assert r1 == r2 and tr.same_bits(b1, b2), (kind, lay, aligned, r1, r2)
                assert "_epi" not in r2[1]


# ==== 7. the tensor-level interface =================================================================================
@gpu
@pytest.mark.parametrize("ind", ["float16", "bfloat16"])
def test_python_gemm_linear(gemm, ind):
    """gemm(x, W.t(), bias=b, activation=a) is act(F.linear(x, W, b)): within the 16-bit tolerance of check_ref16 (an
    activation's slope is at most 1.13) of the float64 answer, for fp32 and 16-bit C, in one launch of the NT _epi
    kernel, without a copy of W."""
    import torch.nn.functional as F
    g = torch.Generator(device="cuda").manual_seed(1800)
    d = dt(ind)
    x = (torch.rand((300, 520), device="cuda", generator=g) * 2 - 1).to(d)
    W = (torch.rand((264, 520), device="cuda", generator=g) * 2 - 1).to(d)
    b = (torch.rand(264, device="cuda", generator=g) * 2 - 1).to(d)
    fns = {None: lambda t: t, "relu": F.relu, "gelu": F.gelu, "gelu_tanh": lambda t: F.gelu(t, approximate="tanh")}
    t64 = F.linear(x.double(), W.double(), b.double())
    scale = float((x.double().abs() @ W.double().abs().t()).max()) + float(b.double().abs().max())
    for act, fn in fns.items():
        want = fn(t64)
        for cd in (torch.float32, d):
            before = gemm.launch_count()
            got = gemm.gemm(x, W.t(), bias=b, activation=act, out_dtype=cd)
            assert gemm.launch_count() - before == 1 and got.dtype == cd
            prefix = {"float16": "tc_f16", "bfloat16": "tc_bf16"}[ind] + ("" if cd == torch.float32 else
                                                                          {"float16": "_of16", "bfloat16": "_obf16"}[ind])
            assert gemm.last_kernel() == f"{prefix}_epi_nt_128x128", gemm.last_kernel()
            rel = {torch.float32: 0.0, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}[cd]
            err = (got.double() - want).abs() - want.abs() * rel
            assert float(err.max()) <= 1.13 * ts.TOL["bf16"] * scale, (ind, act, cd, float(err.max()) / scale)
    # bias only, and activation only
    got = gemm.gemm(x, W.t(), bias=b)
    assert tr.same_bits(got, gemm.gemm(x, W.t(), bias=b, activation=None))
    out = torch.empty((300, 264), device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    gemm.gemm(x, W.t(), out=out, activation="relu")
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() == before                  # no copy of W or of C
    assert tr.same_bits(out, torch.relu(gemm.gemm(x, W.t())))
