"""FP8 outputs of the FP8 GEMMs (b200_gemm_fp8_q8, b200_gemm_fp8_blockwise_q8), scaled_mm(out_dtype=float8_*,
scale_result=...) and scaled_mm_quant().

Each element's fp32 value v is what the fp32-output call on the same inputs stores (the bf16 bias passed as fp32 values),
followed by the activation.  So the oracle is exact: C32 = that call, v = act(C32) (numpy for ReLU, the device's own
epi_act through the bf16 gemm epilogue for the GELUs), and then
  static:   c = fp8(rn(v / s_r))
  dynamic:  d = rn(amax / F) per row and 128-column block (1 when 0, NaN for a NaN / inf block), c = fp8(rn(v / d))
with fp8() round to nearest even and finite values saturated.  Every FP8 output must equal it bit for bit.

The argument checks, the Python refusals and recipe resolution, and the numpy quantiser against torch's CPU casts need
no GPU."""
import numpy as np
import pytest

from test_fp8_gpu import (E4M3, E5M2, OP_N, OP_T, OUT_F32, PAIR_NAME, PAIRS, _has_gpu, decode, encode, exact_operands,
                          fp8_dtype, pow2_scales)
from test_fp8_blockwise_gpu import MAX_INDEX, RECIPE_NAME, RECIPES, cdiv, random_scales, recipe_scales

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")
CT_NAME = {E4M3: "oe4m3", E5M2: "oe5m2"}
SC_SENTINEL = 0x7F7FA5A5     # scale_c fence: a finite fp32 (about 3.4e38) above every scale d = amax / F can take
FMAX = {E4M3: np.float32(448.0), E5M2: np.float32(57344.0)}
ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3
ACT_NAME = {ACT_NONE: None, ACT_RELU: "relu", ACT_GELU: "gelu", ACT_GELU_TANH: "gelu_tanh"}
# input recipes: ("row", fast, bn) tensorwise / rowwise, or ("blk", (a_blk, b_blk))
INPUTS = [("tensor", 0, 0), ("row", 0, 0), ("row", 1, 256), ("row", 1, 128)] + [("blk", b, 0) for b in RECIPES]
INPUT_NAME = lambda r: (f"{r[0]}-{'fast' + str(r[2]) if r[1] else 'promoted'}" if r[0] != "blk" else  # noqa: E731
                        "blk-" + RECIPE_NAME[r[1]])


# ==== the numpy quantiser (the oracle's last step) ==================================================================
def fp8_sat(y, ct):
    """float32 -> FP8 bytes, round to nearest even with finite values saturated to +-F (cvt.rn.satfinite)."""
    with np.errstate(invalid="ignore"):
        return encode(np.clip(np.asarray(y, np.float32), -FMAX[ct], FMAX[ct]), ct)


def quant_static(v, ct, s_r=1.0):
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return fp8_sat((v / np.float32(s_r)).astype(np.float32), ct)


def quant_dynamic(v, ct):
    """(bytes, d): the 1 x 128 quantisation of v (m x n float32)."""
    m, n = v.shape
    qn = cdiv(n, 128)
    vp = np.zeros((m, qn * 128), np.float32)
    vp[:, :n] = v
    blocks = vp.reshape(m, qn, 128)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        bad = ~np.isfinite(blocks).all(axis=2)
        amax = np.where(np.isfinite(blocks), np.abs(blocks), 0).max(axis=2).astype(np.float32)
        d = (amax / FMAX[ct]).astype(np.float32)
        d[d == 0] = 1
        d[bad] = np.nan
        y = (v / np.repeat(d, 128, axis=1)[:, :n]).astype(np.float32)
    return fp8_sat(y, ct), d


def same_fp8(x, y, ct):
    """Same bytes, or NaN at the same places."""
    fx, fy = decode(x, ct), decode(y, ct)
    nx, ny = np.isnan(fx), np.isnan(fy)
    return np.array_equal(nx, ny) and np.array_equal(np.where(nx, 0, x), np.where(ny, 0, y))


def same_f32(x, y):
    nx, ny = np.isnan(x), np.isnan(y)
    return np.array_equal(nx, ny) and np.array_equal(np.where(nx, 0, x).view(np.uint32), np.where(ny, 0, y).view(np.uint32))


@need_torch
def test_quantiser_matches_torch_casts_in_range():
    """fp8_sat is torch's CPU cast on in-range values (rounding included); past +-F it saturates."""
    rng = np.random.default_rng(2)
    for ct in (E4M3, E5M2):
        x = (rng.standard_normal(20000) * float(FMAX[ct]) / 4).astype(np.float32)
        x = x[np.abs(x) <= FMAX[ct]]
        assert np.array_equal(fp8_sat(x, ct), encode(x, ct))
        assert decode(fp8_sat(np.float32([1e30, -1e30, np.inf]), ct), ct).tolist() == \
            [float(FMAX[ct]), -float(FMAX[ct]), float(FMAX[ct])]
        q, d = quant_dynamic(np.float32([[0.0, 0.0], [1.0, -2.0], [np.nan, 1.0]]), ct)
        assert d[0, 0] == 1 and d[1, 0] == np.float32(2.0) / FMAX[ct] and np.isnan(d[2, 0])
        assert decode(q[1], ct)[1] == -float(FMAX[ct])


# ==== the C ABI through ctypes =====================================================================================
def call(gemm, op_a=OP_N, op_b=OP_T, ta=E4M3, tb=E4M3, m=4, n=4, k=4, a=1, lda=None, b=1, ldb=None, sa=1, sa_row=0,
         sb=1, sb_col=0, bias=None, act=0, fast=0, ct=E4M3, c=1, ldc=None, sr=None, scale_c=None, sc_row=None,
         sc_blk=1):
    lda = lda if lda is not None else (m if op_a else k)
    ldb = ldb if ldb is not None else (k if op_b else n)
    ldc = ldc if ldc is not None else n
    sc_row = sc_row if sc_row is not None else cdiv(n, 128)
    return gemm.lib.b200_gemm_fp8_q8(op_a, op_b, ta, tb, m, n, k, a, lda, b, ldb, sa, sa_row, sb, sb_col, bias, act, fast,
                                     ct, c, ldc, sr, scale_c, sc_row, sc_blk, None)


def call_blk(gemm, op_a=OP_N, op_b=OP_T, ta=E4M3, tb=E4M3, m=4, n=4, k=4, a=1, lda=None, b=1, ldb=None, sa=1, a_blk=1,
             sb=1, b_blk=128, bias=None, act=0, ct=E4M3, c=1, ldc=None, sr=None, scale_c=None, sc_row=None, sc_blk=1,
             sa_row=None, sa_kb=1, sb_kb=None, sb_col=1):
    lda = lda if lda is not None else (m if op_a else k)
    ldb = ldb if ldb is not None else (k if op_b else n)
    ldc = ldc if ldc is not None else n
    q = cdiv(k, 128)
    sa_row = sa_row if sa_row is not None else q
    sb_kb = sb_kb if sb_kb is not None else (cdiv(n, 128) if b_blk == 128 else n)
    sc_row = sc_row if sc_row is not None else cdiv(n, 128)
    return gemm.lib.b200_gemm_fp8_blockwise_q8(op_a, op_b, ta, tb, m, n, k, a, lda, b, ldb, sa, a_blk, sa_row, sa_kb, sb,
                                               b_blk, sb_kb, sb_col, bias, act, ct, c, ldc, sr, scale_c, sc_row, sc_blk,
                                               None)


def test_q8_argument_validation(gemm):
    """Refusals before the device is touched, each at its exact bound: they hold with or without a GPU."""
    for f in (call, call_blk):
        assert f(gemm, ct=2) == -1 and f(gemm, ct=-1) == -1 and f(gemm, ct=3) == -1
        assert f(gemm, act=4) == -1 and f(gemm, act=-1) == -1
        assert f(gemm, ta=2) == -1 and f(gemm, tb=-1) == -1
        assert f(gemm, scale_c=1, sr=1) == -1                               # one mode or the other
        assert f(gemm, scale_c=1, sc_row=-1) == -1 and f(gemm, scale_c=1, sc_blk=-1) == -1
        assert f(gemm, op_a=2) == -1 and f(gemm, m=-1) == -1 and f(gemm, k=-1) == -1
        assert f(gemm, m=5, n=6, k=7, ldc=5) == -1                          # ldc >= n bytes
        assert f(gemm, a=None) == -1 and f(gemm, c=None) == -1 and f(gemm, sa=None) == -1 and f(gemm, sb=None) == -1
        assert f(gemm, ta=E5M2, tb=E5M2) == -3
        assert f(gemm, m=0, a=None, b=None, c=None, sa=None, sb=None) == 0
        assert f(gemm, n=0, a=None, b=None, c=None, sa=None, sb=None) == 0
        assert f(gemm, m=0, ct=2) == -1
        # scale_c layouts that could overlap (m = 4, n = 300: q_n = 3)
        for sc_row, sc_blk in ((2, 1), (3, 0), (1, 3), (0, 4), (3, 3), (4, 2)):
            assert f(gemm, m=4, n=300, scale_c=1, sc_row=sc_row, sc_blk=sc_blk) == -1, (sc_row, sc_blk)
        assert f(gemm, m=4, n=300, scale_c=1, sc_row=MAX_INDEX, sc_blk=1) == -1   # last index past the bound
    assert call(gemm, fast=2) == -1 and call(gemm, sa_row=2) == -1
    assert call_blk(gemm, a_blk=128, b_blk=128) == -3 and call_blk(gemm, a_blk=2) == -1
    # b200_gemm_fp8 keeps refusing an FP8 out_type
    assert gemm.lib.b200_gemm_fp8(OP_N, OP_T, E4M3, E4M3, 4, 4, 4, 1, 4, 1, 4, 1, 0, 1, 0, None, 1, 4, 3, 0, None) == -1


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_q8_accepts_at_the_bounds_without_device(gemm):
    """Legal calls at the bounds reach the device check (-2)."""
    for f in (call, call_blk):
        for ct in (E4M3, E5M2):
            for act in range(4):
                assert f(gemm, ct=ct, act=act) == -2
                assert f(gemm, ct=ct, act=act, scale_c=1) == -2
                assert f(gemm, ct=ct, act=act, sr=1) == -2
        for ta, tb in PAIRS:
            assert f(gemm, ta=ta, tb=tb) == -2
        for sc_row, sc_blk in ((3, 1), (9, 1), (1, 4), (1, 9)):              # m = 4, q_n = 3: both layouts, padded
            assert f(gemm, m=4, n=300, scale_c=1, sc_row=sc_row, sc_blk=sc_blk) == -2, (sc_row, sc_blk)
        assert f(gemm, m=1, n=300, scale_c=1, sc_row=0, sc_blk=1) == -2       # extent-1 rows: the row stride is free
        assert f(gemm, m=4, n=100, scale_c=1, sc_row=1, sc_blk=0) == -2       # one block: the block stride is free
        assert f(gemm, m=2, n=300, scale_c=1, sc_row=MAX_INDEX - 2, sc_blk=1) == -2
        assert f(gemm, k=0, a=None, b=None) == -2
        assert f(gemm, m=5, n=6, k=7, ldc=6) == -2
        for op_a in (OP_N, OP_T):
            for op_b in (OP_N, OP_T):
                assert f(gemm, op_a, op_b, m=5, n=6, k=7) == -2
    for fast in (0, 1):
        assert call(gemm, fast=fast, sa_row=1, sb_col=1) == -2


# ==== Python: refusals and resolution (CPU) ========================================================================
def _fp8(shape, t=E4M3):
    return torch.zeros(shape, dtype=torch.float32).to(fp8_dtype(t))


@need_torch
def test_python_refusals_and_resolution(gemm):
    m, n, k = 200, 300, 401
    q, nb = 4, 3
    A, B = _fp8((m, k)), _fp8((k, n))
    one = torch.ones(1)
    # resolved recipes reach the CUDA check; an FP8 out_dtype goes to the FP8-output path
    for sa, sb in ((one, one), (torch.ones(m, 1), torch.ones(1, n)), (torch.ones(m, q), torch.ones(q, nb))):
        for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
            with pytest.raises(ValueError, match="CUDA"):
                gemm.scaled_mm(A, B, sa, sb, out_dtype=dt, scale_result=torch.ones(()))
            with pytest.raises(ValueError, match="CUDA"):
                gemm.scaled_mm_quant(A, B, sa, sb, out_dtype=dt, activation="gelu")
    with pytest.raises(ValueError, match="scale_result"):
        gemm.scaled_mm(A, B, one, one, scale_result=torch.ones(()))          # bf16 output
    with pytest.raises(ValueError, match="scale_result"):
        gemm.scaled_mm(A, B, one, one, out_dtype=torch.float8_e4m3fn, scale_result=torch.ones(2))
    with pytest.raises(ValueError, match="bfloat16"):
        gemm.scaled_mm(A, B, one, one, out_dtype=torch.float8_e4m3fn, bias=torch.zeros(n))
    with pytest.raises(ValueError, match="activation"):
        gemm.scaled_mm_quant(A, B, one, one, activation="tanh")
    with pytest.raises(ValueError, match="use_fast_accum"):
        gemm.scaled_mm_quant(A, B, torch.ones(m, q), torch.ones(q, nb), use_fast_accum=True)
    with pytest.raises(ValueError, match="out_scale"):
        gemm.scaled_mm_quant(A, B, one, one, out_scale=torch.ones(m, nb + 1))
    with pytest.raises(ValueError, match="out_scale"):
        gemm.scaled_mm_quant(A, B, one, one, out_scale=torch.ones(m, nb, dtype=torch.float64))
    with pytest.raises(ValueError, match="out_scale"):                    # overlapping rows
        gemm.scaled_mm_quant(A, B, one, one, out_scale=torch.ones(m * nb).as_strided((m, nb), (2, 1)))
    with pytest.raises(ValueError, match="out_dtype"):
        gemm.scaled_mm_quant(A, B, one, one, out_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="out must"):
        gemm.scaled_mm_quant(A, B, one, one, out_dtype=torch.float8_e4m3fn, out=torch.empty(m, n, dtype=torch.float8_e5m2))
    with pytest.raises(TypeError):
        gemm.scaled_mm_quant(_fp8((m, k), E5M2), _fp8((k, n), E5M2), one, one)
    for out_scale in (torch.ones(m, nb), torch.ones(nb, m).t()):           # both layouts pass to the CUDA check
        with pytest.raises(ValueError, match="CUDA"):
            gemm.scaled_mm_quant(A, B, one, one, out_scale=out_scale)


# ==== GPU ==========================================================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def bf16_values(rng, n):
    """n bf16-representable float32 values (the bias), zeros of both signs included."""
    v = torch.from_numpy((rng.standard_normal(n) * 4).astype(np.float32)).bfloat16().float().numpy()
    v[:2] = [0.0, -0.0][: min(n, 2)]
    return v


class Case:
    """One input recipe on device operands (N, T): C32 (fp32 output, bias as fp32) and the FP8-output calls."""

    def __init__(self, gemm, recipe, ta, tb, m, n, k, rng, exact=False, bias=True):
        self.gemm, self.recipe, self.ta, self.tb, self.m, self.n, self.k = gemm, recipe, ta, tb, m, n, k
        if exact:
            self.a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        else:
            self.a8 = encode(rng.standard_normal((m, k)) * 2, ta)
            b8 = encode(rng.standard_normal((k, n)) * 2, tb)
        self.bt8 = np.ascontiguousarray(b8.T)                            # (n, k)
        self.A, self.Bt = dev(self.a8), dev(self.bt8)
        kind = recipe[0]
        if kind == "blk":
            sa, sb = recipe_scales(rng, recipe[1], m, n, k)
            self.Sa, self.Sb = dev(sa), dev(sb)
        else:
            rows = kind == "row"
            self.Sa = dev(random_scales(rng, (m if rows else 1,)))
            self.Sb = dev(random_scales(rng, (n if rows else 1,)))
        self.bias = bf16_values(rng, n) if bias else None
        self.Bi16 = torch.from_numpy(self.bias).bfloat16().cuda() if bias else None
        self.Bi32 = dev(self.bias) if bias else None

    def _args(self, A=None, lda=None, Bt=None, ldb=None, op_a=OP_N, op_b=OP_T):
        A = self.A if A is None else A
        Bt = self.Bt if Bt is None else Bt
        return (op_a, op_b, self.ta, self.tb, self.m, self.n, self.k, A.data_ptr(), lda or self.k, Bt.data_ptr(),
                ldb or self.k)

    def _scales(self):
        if self.recipe[0] == "blk":
            ab, bb = self.recipe[1]
            return (self.Sa.data_ptr(), ab, *self.Sa.stride(), self.Sb.data_ptr(), bb, *self.Sb.stride())
        return (self.Sa.data_ptr(), int(self.Sa.numel() > 1), self.Sb.data_ptr(), int(self.Sb.numel() > 1))

    def _bn(self):
        self.gemm.lib.b200_gemm_debug_set_bn(self.recipe[2] if self.recipe[0] != "blk" and self.recipe[1] else 0)

    def c32(self):
        m, n = self.m, self.n
        C = torch.full((m, n), float("nan"), dtype=torch.float32, device="cuda")
        bi = self.Bi32.data_ptr() if self.Bi32 is not None else None
        self._bn()
        if self.recipe[0] == "blk":
            rc = self.gemm.lib.b200_gemm_fp8_blockwise(*self._args(), *self._scales(), bi, C.data_ptr(), n, OUT_F32, None)
        else:
            rc = self.gemm.lib.b200_gemm_fp8(*self._args(), *self._scales(), bi, C.data_ptr(), n, OUT_F32,
                                             self.recipe[1], None)
        self.gemm.lib.b200_gemm_debug_set_bn(0)
        assert rc == 0, rc
        torch.cuda.synchronize()
        return C.cpu().numpy()

    def q8(self, ct, act=ACT_NONE, sr=None, dynamic=False, ldc=None, pad=0, sc_layout="row", args=None):
        """The FP8-output call; C (and scale_c) inside sentinel-filled buffers, checked untouched outside."""
        m, n = self.m, self.n
        ldc = ldc or n
        qn = cdiv(n, 128)
        Cbuf = torch.full((pad + m * ldc + pad,), 0xA5, dtype=torch.uint8, device="cuda")
        Cp = Cbuf.data_ptr() + pad
        # scale_c inside 8 fence floats on each side, all of a finite bit pattern no scale can take (d <= 2^128 / 448)
        Sbuf = torch.full((8 + m * qn + 8,), SC_SENTINEL, dtype=torch.int32, device="cuda")
        if sc_layout == "row":
            sc_row, sc_blk = qn, 1
        else:
            sc_row, sc_blk = 1, m
        Sr = dev(np.float32([sr])) if sr is not None else None
        bi = self.Bi16.data_ptr() if self.Bi16 is not None else None
        out = (ct, Cp, ldc, Sr.data_ptr() if Sr is not None else None,
               Sbuf.data_ptr() + 4 * 8 if dynamic else None, sc_row, sc_blk, None)
        self._bn()
        if self.recipe[0] == "blk":
            rc = self.gemm.lib.b200_gemm_fp8_blockwise_q8(*(args or self._args()), *self._scales(), bi, act, *out)
        else:
            rc = self.gemm.lib.b200_gemm_fp8_q8(*(args or self._args()), *self._scales(), bi, act, self.recipe[1], *out)
        self.gemm.lib.b200_gemm_debug_set_bn(0)
        assert rc == 0, rc
        torch.cuda.synchronize()
        self.kernel = self.gemm.last_kernel()
        cb = Cbuf.cpu().numpy()
        body = cb[pad:pad + m * ldc].reshape(m, ldc)
        assert (cb[:pad] == 0xA5).all() and (cb[pad + m * ldc:] == 0xA5).all() and (body[:, n:] == 0xA5).all()
        C = np.ascontiguousarray(body[:, :n])
        sb = Sbuf.cpu().numpy()
        assert (sb[:8] == SC_SENTINEL).all() and (sb[8 + m * qn:] == SC_SENTINEL).all()   # nothing written outside
        if not dynamic:
            return C, None
        assert not (sb[8:8 + m * qn] == SC_SENTINEL).any()                                # every scale written
        s = sb[8:8 + m * qn].view(np.float32)
        d = s.reshape(m, qn) if sc_layout == "row" else s.reshape(qn, m).T
        return C, np.ascontiguousarray(d)


def relu_np(x):
    return np.where(x < 0, np.float32(0), x).astype(np.float32)


def act_dev(gemm, x, act):
    """act(x) by the device's own epilogue (epi_act): the bf16 gemm with zero operands, beta = 1 and fp32 C."""
    m, n = x.shape
    C = dev(x.astype(np.float32))
    Z = torch.zeros((m, 16), dtype=torch.bfloat16, device="cuda")
    W = torch.zeros((16, n), dtype=torch.bfloat16, device="cuda")
    gemm.gemm(Z, W, out=C, beta=1.0, activation=ACT_NAME[act])
    torch.cuda.synchronize()
    return C.cpu().numpy()


def same_or_both_zero(got, want, ct):
    """Same bytes elementwise, or both NaN, or both zero of either sign."""
    fg, fw = decode(got, ct), decode(want, ct)
    return bool(np.all((got == want) | (np.isnan(fg) & np.isnan(fw)) | ((fg == 0) & (fw == 0))))


@gpu
@pytest.mark.parametrize("recipe", INPUTS, ids=INPUT_NAME)
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: PAIR_NAME[p])
@pytest.mark.parametrize("ct", [E4M3, E5M2], ids=lambda c: CT_NAME[c])
def test_cross_path_bit_identity(gemm, recipe, pair, ct):
    """The main gate: static and dynamic outputs equal fp8(C32 / s_r) and the numpy 1 x 128 quantisation of C32, bit for
    bit, with M / N / K tails, random operands and scales, with and without bias and ReLU."""
    rng = np.random.default_rng(11 + 7 * INPUTS.index(recipe) + 3 * PAIRS.index(pair) + ct)
    for m, n, k in ((130, 1, 200), (77, 127, 128), (129, 128, 300), (200, 129, 64), (150, 300, 416)):
        case = Case(gemm, recipe, *pair, m, n, k, rng, bias=(n % 2 == 1))
        v = case.c32()
        for act in (ACT_NONE, ACT_RELU):
            va = relu_np(v) if act == ACT_RELU else v
            sr = float(random_scales(rng, (1,))[0])
            got, _ = case.q8(ct, act=act, sr=sr)
            assert same_fp8(got, quant_static(va, ct, sr), ct), (m, n, k, act, "static")
            got, _ = case.q8(ct, act=act)                                   # s_r null = 1
            assert same_fp8(got, quant_static(va, ct), ct), (m, n, k, act, "static 1")
            got, d = case.q8(ct, act=act, dynamic=True)
            wq, wd = quant_dynamic(va, ct)
            assert same_f32(d, wd), (m, n, k, act, "scales")
            assert same_fp8(got, wq, ct), (m, n, k, act, "dynamic")
        name = f"tc_{PAIR_NAME[pair]}_{CT_NAME[ct]}_"
        if recipe[0] == "blk":
            assert case.kernel == name + "blk_128x128"
        elif recipe[1]:
            assert case.kernel == name + f"128x{recipe[2]}"
        else:
            assert case.kernel == name + "acc_128x128"


@gpu
@pytest.mark.parametrize("act", [ACT_GELU, ACT_GELU_TANH], ids=lambda a: ACT_NAME[a])
@pytest.mark.parametrize("recipe", [("row", 0, 0), ("row", 1, 256), ("blk", (1, 128), 0)], ids=INPUT_NAME)
def test_gelu_against_the_device_activation(gemm, act, recipe):
    """The GELUs: v = act(C32) by the device's own epilogue; same bits, or both zero (the oracle's beta step turns -0
    into +0)."""
    rng = np.random.default_rng(21 + act)
    case = Case(gemm, recipe, E4M3, E4M3, 200, 300, 384, rng)
    v = act_dev(gemm, case.c32(), act)
    for ct in (E4M3, E5M2):
        got, _ = case.q8(ct, act=act, sr=0.75)
        assert same_or_both_zero(got, quant_static(v, ct, 0.75), ct)
        got, d = case.q8(ct, act=act, dynamic=True)
        wq, wd = quant_dynamic(v, ct)
        assert same_f32(d, wd)
        assert same_or_both_zero(got, wq, ct)


@gpu
@pytest.mark.parametrize("sc_layout", ["row", "outer"])
def test_chain_into_the_blockwise_gemm(gemm, sc_layout):
    """scaled_mm(*scaled_mm_quant(x, W1^T, ...), W2^T, ...) with a 128 x 128 sW2 equals b200_gemm_fp8_blockwise on the
    numpy-quantised bytes and scales, bit for bit."""
    rng = np.random.default_rng(31)
    m, d, dff = 256, 384, 300
    x8 = encode(rng.standard_normal((m, d)), E4M3)
    w1 = encode(rng.standard_normal((dff, d)), E4M3)
    w2 = encode(rng.standard_normal((d, dff)), E4M3)
    X, W1, W2 = (dev(t).view(torch.float8_e4m3fn) for t in (x8, w1, w2))
    sx, sw1 = dev(random_scales(rng, (m, 1))), dev(random_scales(rng, (1, dff)))
    b1 = torch.from_numpy(bf16_values(rng, dff)).bfloat16().cuda()
    q2 = cdiv(dff, 128)
    sw2 = dev(random_scales(rng, (q2, cdiv(d, 128))))
    out_scale = None if sc_layout == "row" else torch.empty((q2, m), device="cuda").t()
    h, sh = gemm.scaled_mm_quant(X, W1.t(), sx, sw1, bias=b1, activation="relu", out_scale=out_scale)
    assert h.dtype == torch.float8_e4m3fn and sh.shape == (m, q2)
    y = gemm.scaled_mm(h, W2.t(), sh, sw2, out_dtype=torch.float32)
    # the oracle: C32 of layer 1, numpy quantisation, then the blockwise call on those bytes and scales
    v = relu_np(gemm.scaled_mm(X, W1.t(), sx, sw1, bias=b1.float(), out_dtype=torch.float32).cpu().numpy())
    hq, hd = quant_dynamic(v, E4M3)
    assert np.array_equal(h.view(torch.uint8).cpu().numpy(), hq) and same_f32(sh.cpu().numpy(), hd)
    want = gemm.scaled_mm(dev(hq).view(torch.float8_e4m3fn), W2.t(), dev(hd), sw2, out_dtype=torch.float32)
    assert same_f32(y.cpu().numpy(), want.cpu().numpy())


def torch_fp8_out_combos():
    for ta, tb in PAIRS:
        for ct in (E4M3, E5M2):
            yield ta, tb, ct


@gpu
@pytest.mark.parametrize("combo", list(torch_fp8_out_combos()), ids=lambda c: f"{PAIR_NAME[c[:2]]}-{CT_NAME[c[2]]}")
def test_against_torch_scaled_mm(gemm, combo):
    """torch._scaled_mm with an FP8 out (tensorwise scales, every combination torch accepts): equal bits on integer
    operands with power-of-two scales, within one FP8 ulp on random operands, and the same saturation on overflow.
    torch on CUDA ignores scale_result in this build (DESIGN §9), so the comparison passes none."""
    ta, tb, ct = combo
    rng = np.random.default_rng(41)
    m, n, k = 192, 320, 384
    dt = fp8_dtype(ct)
    for exact in (True, False):
        if exact:
            a8, b8 = exact_operands(rng, m, n, k, ta, tb)
        else:
            a8, b8 = encode(rng.standard_normal((m, k)), ta), encode(rng.standard_normal((k, n)), tb)
        A = dev(a8).view(fp8_dtype(ta))
        W = dev(np.ascontiguousarray(b8.T)).view(fp8_dtype(tb))
        sa, sb = dev(pow2_scales(rng, 1).reshape(())), dev(pow2_scales(rng, 1).reshape(()))
        bias = torch.from_numpy(rng.integers(-8, 9, n).astype(np.float32) / 4).bfloat16().cuda()
        for bi in (None, bias):
            try:
                want = torch._scaled_mm(A, W.t(), sa, sb, bias=bi, out_dtype=dt)
            except (RuntimeError, NotImplementedError) as e:
                pytest.skip(f"torch._scaled_mm refuses this combination: {str(e).splitlines()[0]}")
            got = gemm.scaled_mm(A, W.t(), sa, sb, bias=bi, out_dtype=dt)
            g, w = got.view(torch.uint8).cpu().numpy(), want.view(torch.uint8).cpu().numpy()
            if exact:
                assert np.array_equal(g, w), bi is None
            else:                           # one ulp: adjacent codes of the same sign (or +-0)
                gi, wi = g.astype(np.int16), w.astype(np.int16)
                same_sign = (gi & 0x80) == (wi & 0x80)
                assert bool(np.all((same_sign & (np.abs(gi - wi) <= 1)) | ((gi & 0x7F) + (wi & 0x7F) <= 1)))
    # overflow: both saturate to +-F
    big = torch.full((32, 64), 128.0).to(fp8_dtype(ta)).cuda()
    for sign in (1.0, -1.0):
        Wb = torch.full((32, 64), 128.0 * sign).to(fp8_dtype(tb)).cuda()
        one = torch.ones((), device="cuda")
        try:
            want = torch._scaled_mm(big, Wb.t(), one, one, out_dtype=dt)
        except (RuntimeError, NotImplementedError) as e:
            pytest.skip(f"torch._scaled_mm refuses this combination: {str(e).splitlines()[0]}")
        got = gemm.scaled_mm(big, Wb.t(), one, one, out_dtype=dt)
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
        assert got.float()[0, 0].item() == sign * float(FMAX[ct])


@gpu
@pytest.mark.parametrize("ct", [E4M3, E5M2], ids=lambda c: CT_NAME[c])
def test_non_finite_zero_and_underflow_blocks(gemm, ct):
    """A NaN or inf scale or operand makes its blocks NaN (d = NaN), an all-zero block has d = 1, an underflowing block
    (amax / F rounds to 0) too; the static mode keeps NaN and saturates inf."""
    rng = np.random.default_rng(51)
    m, n, k = 130, 300, 256
    for recipe in (("row", 0, 0), ("row", 1, 256), ("blk", (1, 128), 0)):
        case = Case(gemm, recipe, E4M3, E4M3, m, n, k, rng, exact=True, bias=False)
        a8 = case.a8.copy()
        a8[3, :] = 0                                                       # row 3: all-zero blocks
        a8[5, 7] = 0x7F                                                    # row 5: NaN operand (all blocks)
        case.A = dev(a8)
        if recipe[0] == "blk":
            sb = case.Sb.cpu().numpy()
            sb[0, 1] = np.inf                                               # column block 1, k-block 0: inf scale
            case.Sb = dev(sb)
            sa = case.Sa.cpu().numpy()
            sa[9, :] = 1e-45                                                # row 9: underflow
            case.Sa = dev(sa)
        else:
            sb = case.Sb.cpu().numpy()
            if sb.size > 1:
                sb[200] = np.nan                                            # column block 1: NaN
                case.Sb = dev(sb)
            sa = case.Sa.cpu().numpy()
            if sa.size > 1:
                sa[9] = 1e-45
                case.Sa = dev(sa)
        v = case.c32()
        got, d = case.q8(ct, dynamic=True)
        wq, wd = quant_dynamic(v, ct)
        assert same_f32(d, wd) and same_fp8(got, wq, ct), recipe
        assert d[3, 0] == 1 and np.isnan(d[5]).all()                       # (row 3's block 1 holds the NaN / inf scale)
        got, _ = case.q8(ct, sr=0.5)
        assert same_fp8(got, quant_static(v, ct, 0.5), ct), recipe


@gpu
def test_k_zero_and_empty(gemm):
    """k == 0 quantises v = act(rn(+0 + bias_j)) without reading operands or input scales; m / n == 0 writes nothing."""
    rng = np.random.default_rng(61)
    m, n = 70, 300
    for ct in (E4M3, E5M2):
        for with_bias in (False, True):
            bias = bf16_values(rng, n)
            Bi = torch.from_numpy(bias).bfloat16().cuda() if with_bias else None
            for act in (ACT_NONE, ACT_RELU, ACT_GELU):
                v = np.broadcast_to((np.float32(0) + bias) if with_bias else np.float32(0), (m, n)).astype(np.float32)
                v = act_dev(gemm, v, act) if act else v
                nan = torch.full((m, 2), float("nan"), device="cuda")   # input scales: never read
                for blockwise in (False, True):
                    for dyn in (False, True):
                        C = torch.full((m, n), 0xA5, dtype=torch.uint8, device="cuda")
                        S = torch.full((m, cdiv(n, 128)), float("nan"), device="cuda")
                        bi = Bi.data_ptr() if with_bias else None
                        out = (ct, C.data_ptr(), n, None, S.data_ptr() if dyn else None, S.stride(0), 1, None)
                        if blockwise:
                            rc = gemm.lib.b200_gemm_fp8_blockwise_q8(OP_N, OP_T, E4M3, E4M3, m, n, 0, None, 0, None, 0,
                                                                     nan.data_ptr(), 1, 2, 1, nan.data_ptr(), 128, 0, 0,
                                                                     bi, act, *out)
                        else:
                            rc = gemm.lib.b200_gemm_fp8_q8(OP_N, OP_T, E4M3, E4M3, m, n, 0, None, 0, None, 0,
                                                           nan.data_ptr(), 0, nan.data_ptr(), 0, bi, act, 0, *out)
                        assert rc == 0
                        torch.cuda.synchronize()
                        got = C.cpu().numpy()
                        if dyn:
                            wq, wd = quant_dynamic(v, ct)
                            assert same_f32(S.cpu().numpy(), wd)
                        else:
                            wq = quant_static(v, ct)
                        assert same_or_both_zero(got, wq, ct) if act else same_fp8(got, wq, ct)
        for mm, nn in ((0, n), (m, 0)):
            C = torch.full((m, n), 7, dtype=torch.uint8, device="cuda")
            rc = gemm.lib.b200_gemm_fp8_q8(OP_N, OP_T, E4M3, E4M3, mm, nn, 16, None, 16, None, 16, None, 0, None, 0, None, 0,
                                           0, ct, C.data_ptr(), n, None, None, 0, 0, None)
            assert rc == 0 and bool((C == 7).all())


@gpu
@pytest.mark.parametrize("recipe", [("row", 0, 0), ("row", 1, 128), ("blk", (1, 1), 0)], ids=INPUT_NAME)
def test_layouts_pitches_and_odd_ldc(gemm, recipe):
    """NN / TN / TT and unaligned pitches give the (N, T) bits; an odd ldc and an odd C base work."""
    rng = np.random.default_rng(71)
    m, n, k = 150, 260, 200
    case = Case(gemm, recipe, E4M3, E5M2, m, n, k, rng)
    ref, ref_d = case.q8(E4M3, dynamic=True)
    a8, bt8 = case.a8, case.bt8
    b8 = np.ascontiguousarray(bt8.T)
    for op_a in (OP_N, OP_T):
        for op_b in (OP_N, OP_T):
            for extra in (0, 3):
                sa_ = np.ascontiguousarray(a8.T) if op_a else a8
                sb_ = bt8 if op_b else b8
                pa = np.zeros((sa_.shape[0], sa_.shape[1] + extra), np.uint8)
                pa[:, :sa_.shape[1]] = sa_
                pb = np.zeros((sb_.shape[0], sb_.shape[1] + extra), np.uint8)
                pb[:, :sb_.shape[1]] = sb_
                A, B = dev(pa), dev(pb)
                args = (op_a, op_b, case.ta, case.tb, m, n, k, A.data_ptr(), pa.shape[1], B.data_ptr(), pb.shape[1])
                got, d = case.q8(E4M3, dynamic=True, args=args)
                assert np.array_equal(got, ref) and same_f32(d, ref_d), (op_a, op_b, extra)
    for ldc, pad in ((n + 1, 1), (n + 3, 3), (n, 1)):
        got, d = case.q8(E4M3, dynamic=True, ldc=ldc, pad=pad, sc_layout="outer")
        assert np.array_equal(got, ref) and same_f32(d, ref_d), (ldc, pad)


@gpu
def test_cuda_graph_with_rewritten_scales(gemm):
    """One capture per mode, replayed with scale_a, scale_b and s_r rewritten on the device between replays."""
    rng = np.random.default_rng(81)
    m, n, k = 256, 384, 256
    a8, b8 = exact_operands(rng, m, n, k, E4M3, E4M3)
    A = dev(a8).view(torch.float8_e4m3fn)
    W = dev(np.ascontiguousarray(b8.T)).view(torch.float8_e4m3fn)
    sa, sb = torch.ones((m, 1), device="cuda"), torch.ones((1, n), device="cuda")
    sr = torch.ones((), device="cuda")
    out = torch.empty((m, n), dtype=torch.float8_e4m3fn, device="cuda")
    qout = torch.empty((m, n), dtype=torch.float8_e4m3fn, device="cuda")
    qs = torch.empty((m, 3), device="cuda")
    c32 = torch.empty((m, n), dtype=torch.float32, device="cuda")

    def calls():
        gemm.scaled_mm(A, W.t(), sa, sb, out=out, scale_result=sr)
        gemm.scaled_mm_quant(A, W.t(), sa, sb, out=qout, out_scale=qs)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        calls()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls()
    for _ in range(3):
        sa.copy_(torch.from_numpy(pow2_scales(rng, m)).reshape(m, 1))
        sb.copy_(torch.from_numpy(pow2_scales(rng, n)).reshape(1, n))
        sr.fill_(float(random_scales(rng, (1,))[0]))
        g.replay()
        torch.cuda.synchronize()
        gemm.scaled_mm(A, W.t(), sa, sb, out=c32)
        v = c32.cpu().numpy()
        assert np.array_equal(out.view(torch.uint8).cpu().numpy(), quant_static(v, E4M3, sr.item()))
        wq, wd = quant_dynamic(v, E4M3)
        assert np.array_equal(qout.view(torch.uint8).cpu().numpy(), wq) and same_f32(qs.cpu().numpy(), wd)


@gpu
def test_mlp_sized_gelu_dynamic(gemm):
    """An MLP-sized call, 2048 x 14336 x 4096 with GELU in dynamic mode, equals the quantisation of act(C32)."""
    rng = np.random.default_rng(91)
    m, n, k = 2048, 14336, 4096
    x = torch.from_numpy(rng.standard_normal((m, k)).astype(np.float32)).cuda()
    Wf = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).cuda()
    sx = (x.abs().amax(dim=1, keepdim=True) / 448).float()
    sw = (Wf.abs().amax(dim=1, keepdim=True) / 448).float()
    xq, wq = (x / sx).to(torch.float8_e4m3fn), (Wf / sw).to(torch.float8_e4m3fn)
    del x, Wf
    b = torch.from_numpy(bf16_values(rng, n)).bfloat16().cuda()
    h, sh = gemm.scaled_mm_quant(xq, wq.t(), sx, sw.t(), bias=b, activation="gelu")
    c32 = gemm.scaled_mm(xq, wq.t(), sx, sw.t(), bias=b.float(), out_dtype=torch.float32)
    v = act_dev(gemm, c32.cpu().numpy(), ACT_GELU)
    wq_, wd = quant_dynamic(v, E4M3)
    assert same_f32(sh.cpu().numpy(), wd)
    assert same_or_both_zero(h.view(torch.uint8).cpu().numpy(), wq_, E4M3)
